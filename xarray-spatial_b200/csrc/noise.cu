// noise.cu -- perlin (perlin.py:189) and generate_terrain (terrain.py:183) on the device, with the reference's
// NumPy path as the semantics (DESIGN.md section 4.10).
//
// xrs_perm_tables builds RandomState(seed).permutation(n) for every seed of a call on the device: MT19937 word
// streams (one CTA per seed), the rejection draws resolved 32 words at a time (one warp per seed), then the
// Fisher-Yates swaps applied by the deterministic reservations of Shun et al. (SODA 2015), round by round from the
// host.  xrs_noise evaluates the octaves from per-column and per-row tables, fuses all octaves of a cell, and
// normalises in an epilogue.  The arithmetic shared with the CPU tests sits in noise_octave.cuh.
#include <math.h>

#include <algorithm>

#include "common.cuh"
#include "noise_octave.cuh"

namespace xrs {
namespace {

using namespace nz;

constexpr int kMaxSeeds = 32;
constexpr int kGenThreads = 640;                  // one per state word, rounded up to whole warps
constexpr int kResolveUnroll = 16;                // words per lane in flight in the resolve
constexpr int64_t kChunkBlocks = 832;             // 624-word blocks per generated chunk
constexpr int64_t kChunk = kChunkBlocks * kMtN;   // 519168 words, a multiple of 32 * kResolveUnroll
constexpr int kFirstChunks = 3;                   // 1.56 M words: a 2^20 table draws about 1.45 M
constexpr int kMaxChunks = 64;
constexpr int kBatch = 8;                         // shuffle rounds enqueued between two reads of the counts
constexpr int64_t kCtl = 256;
static_assert(kChunk % (32 * kResolveUnroll) == 0, "the resolve reads whole groups of words");

struct Seeds {
    uint32_t v[kMaxSeeds];
};

struct TableCtl {
    int count[kBatch + 1];   // pending steps at the start of each round of a batch
};
static_assert(sizeof(TableCtl) <= kCtl, "control block");

struct TableLayout {
    int64_t mt, words, step, J, R, list0, list1, total;
    TableLayout(int S, int64_t n) {
        mt = kCtl;
        words = mt + align256((int64_t)S * kMtN * 4);
        step = words + align256((int64_t)S * kChunk * 4);
        J = step + align256((int64_t)S * 4);
        R = J + align256((int64_t)S * n * 4);
        list0 = R + align256((int64_t)S * n * 8);
        list1 = list0 + align256((int64_t)S * n * 4);
        total = list1 + align256((int64_t)S * n * 4);
    }
};

// Words [chunk kChunk, (chunk + 1) kChunk) of each seed's stream.  The state after the chunk's last twist is kept in
// `state` for the next chunk; chunk 0 starts from init_genrand.  Seeds whose draws are all resolved skip.
__global__ void __launch_bounds__(kGenThreads) nz_gen_kernel(Seeds seeds, uint32_t *state, uint32_t *words,
                                                             int chunk, const uint32_t *step) {
    __shared__ uint32_t mt[kMtN];
    const int s = blockIdx.x, t = threadIdx.x;
    if (step[s] == 0) return;
    if (chunk == 0) {
        if (t == 0) mt_init(mt, seeds.v[s]);
    } else if (t < kMtN) {
        mt[t] = state[s * kMtN + t];
    }
    __syncthreads();
    uint32_t *out = words + (int64_t)s * kChunk;
    for (int64_t b = 0; b < kChunkBlocks; ++b) {
        for (int p = 0; p < 4; ++p) {
            const bool mine = t >= phase_begin(p) && t < phase_begin(p + 1);
            const uint32_t nv = mine ? mt_twist_word(mt, t) : 0;
            __syncthreads();   // every read of the phase before any write
            if (mine) mt[t] = nv;
            __syncthreads();
        }
        if (t < kMtN) out[b * kMtN + t] = mt_temper(mt[t]);
    }
    if (t < kMtN) state[s * kMtN + t] = mt[t];
}

// The draws of one chunk, one warp per seed: step[s] is the next Fisher-Yates step (0 when done) and J receives
// each step's accepted value.  A chunk of 32 words goes through chunk_uniform / sure_accept with two ballots;
// chunks at a change of mask, near the end, or holding an undecided word go word by word.
__global__ void __launch_bounds__(32) nz_resolve_kernel(const uint32_t *words, uint32_t *step, int32_t *J,
                                                        int64_t n) {
    const int s = blockIdx.x, lane = threadIdx.x;
    const unsigned full = 0xffffffffu, below = (1u << lane) - 1u;
    uint32_t i = step[s];
    const uint32_t *w = words + (int64_t)s * kChunk;
    int32_t *Js = J + (int64_t)s * n;
    for (int64_t q = 0; i > 0 && q < kChunk; q += 32 * kResolveUnroll) {
        uint32_t r[kResolveUnroll];
#pragma unroll
        for (int u = 0; u < kResolveUnroll; ++u) r[u] = __ldcs(w + q + 32 * u + lane);
#pragma unroll
        for (int u = 0; u < kResolveUnroll; ++u) {
            if (i == 0) break;
            const uint32_t v = r[u] & interval_mask(i);
            const bool fast = chunk_uniform(i) && !__any_sync(full, undecided(v, i));
            if (fast) {
                const bool acc = sure_accept(v, i);
                const unsigned a = __ballot_sync(full, acc);
                if (acc) Js[i - __popc(a & below)] = (int32_t)v;
                i -= __popc(a);
            } else {
                for (int l = 0; l < 32 && i > 0; ++l) {
                    const uint32_t vl = __shfl_sync(full, r[u], l) & interval_mask(i);
                    if (vl <= i) {
                        if (lane == 0) Js[i] = (int32_t)vl;
                        --i;
                    }
                }
            }
        }
    }
    if (lane == 0) step[s] = i;
}

// A[s][k] = k, and every step i >= 1 of every seed pending (entry s n + i).
__global__ void nz_shuffle_init_kernel(int32_t *A, int32_t *list, int S, int64_t n) {
    const int64_t total = (int64_t)S * n;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t s = e / n, k = e - s * n;
        A[e] = (int32_t)k;
        if (k > 0) list[s * (n - 1) + k - 1] = (int32_t)e;
    }
}

__global__ void nz_reserve_kernel(const int32_t *list, const int *count, const int32_t *J,
                                  unsigned long long *R, int64_t n, uint32_t round) {
    const int m = *count;
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < m; k += gridDim.x * blockDim.x) {
        const int64_t e = list[k], s = e / n, i = e - s * n;
        const unsigned long long key = reservation(round, (uint32_t)i);
        atomicMax(R + e, key);
        atomicMax(R + s * n + J[e], key);
    }
}

__global__ void nz_commit_kernel(const int32_t *list_in, const int *count_in, int32_t *list_out, int *count_out,
                                 const int32_t *J, const unsigned long long *R, int32_t *A, int64_t n,
                                 uint32_t round) {
    const int m = *count_in;
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < m; k += gridDim.x * blockDim.x) {
        const int64_t e = list_in[k], s = e / n, i = e - s * n, j = s * n + J[e];
        const unsigned long long key = reservation(round, (uint32_t)i);
        if (R[e] == key && R[j] == key) {
            const int32_t t = A[e];
            A[e] = A[j];
            A[j] = t;
        } else {
            list_out[atomicAdd(count_out, 1)] = (int32_t)e;
        }
    }
}

int table_args(int n_seeds, int64_t n) {
    XRS_REQUIRE(n_seeds >= 1 && n_seeds <= kMaxSeeds, "n_seeds must be 1 .. 32");
    XRS_REQUIRE(n >= 1 && n <= kTableN, "the table length must be 1 .. 2^20");
    return XRS_OK;
}

// ---------------------------------------------------------------------------------------------- noise
constexpr int kStats = 5;              // per octave: bad coordinate, min P, max P, min yi, max yi
constexpr int kCellThreads = 256;      // 8 warps
constexpr int kUnitRows = 8;           // a warp's unit: 8 rows x 32 columns
constexpr int kMaxCellCtas = 4096;

struct NoiseLayout {
    int64_t result, cols, rows, partials, total;
    NoiseLayout(int64_t H, int64_t W, int n_oct) {
        result = 0;   // the field's min and max before normalisation, as float64 (xrs_b200.h)
        cols = 256;
        rows = cols + align256(n_oct * W * (int64_t)sizeof(Col));
        partials = rows + align256(n_oct * H * (int64_t)sizeof(Row));
        total = partials + align256(kMaxCellCtas * 16);
    }
};

__global__ void nz_stats_init_kernel(int32_t *stats, int n_oct) {
    const int k = threadIdx.x;
    if (k < n_oct * kStats) {
        const int f = k % kStats;
        stats[k] = f == 0 ? 0 : (f == 1 || f == 3) ? INT32_MAX : INT32_MIN;
    }
}

// Octave o's table entries of column j: float32(x 2^o), xi, x - xi, fade, P[xi], P[xi + 1].
__global__ void nz_col_kernel(const int32_t *tables, const float *xs, int64_t W, int n_oct, Col *cols,
                              int32_t *stats) {
    const int64_t total = n_oct * W;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k - threadIdx.x < total;
         k += (int64_t)gridDim.x * blockDim.x) {
        const bool live = k < total;
        const int o = live ? (int)(k / W) : 0;
        bool ok = true;
        Col c{};
        if (live) {
            c = make_col(tables + o * kTableN, octave_coord(xs[k - o * W], o), ok);
            cols[k] = c;
        }
        // the warp's octaves differ only at a boundary; reduce per octave with a match mask
        const unsigned grp = __match_any_sync(0xffffffffu, live ? o : -1);
        const int lo = live && ok ? min(c.p0, c.p1) : INT32_MAX, hi = live && ok ? max(c.p0, c.p1) : INT32_MIN;
        const int mn = __reduce_min_sync(grp, lo), mx = __reduce_max_sync(grp, hi);
        const int bad = __reduce_or_sync(grp, live && !ok);
        if (live && (threadIdx.x & 31) == __ffs(grp) - 1) {
            int32_t *st = stats + o * kStats;
            if (bad) atomicOr(st, 1);
            atomicMin(st + 1, mn);
            atomicMax(st + 2, mx);
        }
    }
}

__global__ void nz_row_kernel(const float *ys, int64_t H, int n_oct, Row *rows, int32_t *stats) {
    const int64_t total = n_oct * H;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k - threadIdx.x < total;
         k += (int64_t)gridDim.x * blockDim.x) {
        const bool live = k < total;
        const int o = live ? (int)(k / H) : 0;
        bool ok = true;
        Row r{};
        if (live) {
            r = make_row(octave_coord(ys[k - o * H], o), ok);
            rows[k] = r;
        }
        const unsigned grp = __match_any_sync(0xffffffffu, live ? o : -1);
        const int mn = __reduce_min_sync(grp, live && ok ? r.yi : INT32_MAX);
        const int mx = __reduce_max_sync(grp, live && ok ? r.yi : INT32_MIN);
        const int bad = __reduce_or_sync(grp, live && !ok);
        if (live && (threadIdx.x & 31) == __ffs(grp) - 1) {
            int32_t *st = stats + o * kStats;
            if (bad) atomicOr(st, 1);
            atomicMin(st + 3, mn);
            atomicMax(st + 4, mx);
        }
    }
}

// np.min / np.max with NaN propagation, as float64 (every cell type widens exactly).
struct MinMax {
    double mn, mx;
    bool nan;
    __device__ void add(double v) {
        if (v != v) nan = true;
        else {
            mn = v < mn ? v : mn;
            mx = v > mx ? v : mx;
        }
    }
    __device__ void merge(const MinMax &o) {
        nan = nan || o.nan;
        mn = o.mn < mn ? o.mn : mn;
        mx = o.mx > mx ? o.mx : mx;
    }
};

__device__ MinMax block_minmax(MinMax m) {
    __shared__ double smn[kCellThreads / 32], smx[kCellThreads / 32];
    __shared__ int snan[kCellThreads / 32];
    for (int d = 16; d > 0; d >>= 1) {
        MinMax o{__shfl_down_sync(0xffffffffu, m.mn, d), __shfl_down_sync(0xffffffffu, m.mx, d),
                 (bool)__shfl_down_sync(0xffffffffu, (int)m.nan, d)};
        m.merge(o);
    }
    const int wid = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) {
        smn[wid] = m.mn;
        smx[wid] = m.mx;
        snan[wid] = m.nan;
    }
    __syncthreads();
    if (threadIdx.x == 0)
        for (int k = 1; k < kCellThreads / 32; ++k) m.merge(MinMax{smn[k], smx[k], (bool)snan[k]});
    return m;
}

// The field before normalisation.  Each warp takes units of 8 rows x 32 columns; per octave a lane loads its
// column's entry once and each row's entry (the same address for the whole warp), then runs octave() per cell.
// perlin (n_oct 1): T(a).  terrain (n_oct 16): h = in 0, h = T(double(h) + a 2^-o) per octave, h / 1.97, cube.
template <typename T, bool TERRAIN>
__global__ void __launch_bounds__(kCellThreads) nz_cell_kernel(const T *in, int64_t in_pitch, int64_t H, int64_t W,
                                                               const int32_t *tables, const Col *cols,
                                                               const Row *rows, int n_oct, T *out,
                                                               int64_t out_pitch, double *partials) {
    const int lane = threadIdx.x & 31;
    const int64_t units_x = (W + 31) / 32, units = units_x * ((H + kUnitRows - 1) / kUnitRows);
    const int64_t warps = (int64_t)gridDim.x * (kCellThreads / 32);
    MinMax m{INFINITY, -INFINITY, false};
    for (int64_t u = (int64_t)blockIdx.x * (kCellThreads / 32) + (threadIdx.x >> 5); u < units; u += warps) {
        const int64_t uy = u / units_x, c = (u - uy * units_x) * 32 + lane, r0 = uy * kUnitRows;
        const int nr = (int)min((int64_t)kUnitRows, H - r0);
        if (c >= W) continue;   // no warp-wide operation below
        T h[kUnitRows];
#pragma unroll
        for (int k = 0; k < kUnitRows; ++k) h[k] = (TERRAIN && k < nr) ? in[(r0 + k) * in_pitch + c] * (T)0 : (T)0;
        for (int o = 0; o < n_oct; ++o) {
            const Col col = cols[o * W + c];
            const int32_t *P = tables + o * kTableN;
            const double mo = octave_weight(o);
#pragma unroll
            for (int k = 0; k < kUnitRows; ++k) {
                if (k < nr) {
                    const double a = octave(P, col, rows[o * H + r0 + k]);
                    h[k] = TERRAIN ? terrain_add(h[k], a, mo) : (T)a;
                }
            }
        }
#pragma unroll
        for (int k = 0; k < kUnitRows; ++k) {
            if (k < nr) {
                const T v = TERRAIN ? terrain_cube(terrain_scale(h[k])) : h[k];
                out[(r0 + k) * out_pitch + c] = v;
                m.add((double)v);
            }
        }
    }
    m = block_minmax(m);
    if (threadIdx.x == 0) {
        partials[2 * blockIdx.x] = m.nan ? nan_of<double>() : m.mn;
        partials[2 * blockIdx.x + 1] = m.nan ? nan_of<double>() : m.mx;
    }
}

__global__ void __launch_bounds__(kCellThreads) nz_minmax_kernel(const double *partials, int n, double *result) {
    MinMax m{INFINITY, -INFINITY, false};
    for (int k = threadIdx.x; k < n; k += kCellThreads) {
        m.add(partials[2 * k]);
        m.add(partials[2 * k + 1]);
    }
    m = block_minmax(m);
    if (threadIdx.x == 0) {
        result[0] = m.nan ? nan_of<double>() : m.mn;
        result[1] = m.nan ? nan_of<double>() : m.mx;
    }
}

template <typename T> __device__ __forceinline__ T sub_rn(T a, T b);
template <> __device__ __forceinline__ float sub_rn<float>(float a, float b) { return __fsub_rn(a, b); }
template <> __device__ __forceinline__ double sub_rn<double>(double a, double b) { return __dsub_rn(a, b); }
template <typename T> __device__ __forceinline__ T div_rn(T a, T b);
template <> __device__ __forceinline__ float div_rn<float>(float a, float b) { return __fdiv_rn(a, b); }
template <> __device__ __forceinline__ double div_rn<double>(double a, double b) { return __ddiv_rn(a, b); }

// (d - min) / (max - min) in T; terrain then sets cells below T(0.3) to 0 and multiplies by T(zfactor).
template <typename T, bool TERRAIN>
__global__ void nz_epilogue_kernel(T *out, int64_t out_pitch, int64_t H, int64_t W, const double *result,
                                   double zfactor) {
    const T mn = (T)result[0], ptp = sub_rn((T)result[1], mn), thr = (T)0.3, zf = (T)zfactor;
    const int64_t n = H * W;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = k / W;
        T *p = out + r * out_pitch + (k - r * W);
        T v = div_rn(sub_rn(*p, mn), ptp);
        if (TERRAIN) {
            if (v < thr) v = (T)0;
            v = v * zf;
        }
        *p = v;
    }
}

int noise_shape(int64_t H, int64_t W) {
    XRS_REQUIRE(H > 0 && W > 0, "the noise functions need a raster of at least one cell");
    XRS_REQUIRE(H < ((int64_t)1 << 31) && W < ((int64_t)1 << 31), "a side of 2^31 cells or more");
    return XRS_OK;
}

template <typename T, bool TERRAIN>
int run_noise(const T *in, int64_t in_pitch, int64_t H, int64_t W, const int32_t *tables, const float *xs,
              const float *ys, double zfactor, T *out, int64_t out_pitch, int32_t *stats, char *scratch,
              const NoiseLayout &L, cudaStream_t s) {
    const int n_oct = TERRAIN ? kTerrainOctaves : 1;
    Col *cols = (Col *)(scratch + L.cols);
    Row *rows = (Row *)(scratch + L.rows);
    double *partials = (double *)(scratch + L.partials), *result = (double *)(scratch + L.result);
    nz_stats_init_kernel<<<1, 128, 0, s>>>(stats, n_oct);
    XRS_CUDA(cudaGetLastError());
    nz_col_kernel<<<(unsigned)stride_grid(n_oct * W), 256, 0, s>>>(tables, xs, W, n_oct, cols, stats);
    XRS_CUDA(cudaGetLastError());
    nz_row_kernel<<<(unsigned)stride_grid(n_oct * H), 256, 0, s>>>(ys, H, n_oct, rows, stats);
    XRS_CUDA(cudaGetLastError());
    const int64_t units = ((W + 31) / 32) * ((H + kUnitRows - 1) / kUnitRows);
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>({(units + 7) / 8, (int64_t)sm_count() * 8,
                                                                   (int64_t)kMaxCellCtas}));
    nz_cell_kernel<T, TERRAIN><<<grid, kCellThreads, 0, s>>>(in, in_pitch, H, W, tables, cols, rows, n_oct, out,
                                                             out_pitch, partials);
    XRS_CUDA(cudaGetLastError());
    nz_minmax_kernel<<<1, kCellThreads, 0, s>>>(partials, grid, result);
    XRS_CUDA(cudaGetLastError());
    nz_epilogue_kernel<T, TERRAIN><<<(unsigned)stride_grid(H * W), 256, 0, s>>>(out, out_pitch, H, W, result,
                                                                                 zfactor);
    XRS_CUDA(cudaGetLastError());
    return XRS_OK;
}

}  // namespace
}  // namespace xrs

using namespace xrs;

extern "C" int xrs_perm_tables_scratch_bytes(int n_seeds, int64_t n, int64_t *bytes) {
    XRS_REQUIRE(bytes != nullptr, "NULL pointer");
    const int rc = table_args(n_seeds, n);
    if (rc) return rc;
    *bytes = TableLayout(n_seeds, n).total;
    return XRS_OK;
}

extern "C" int xrs_perm_tables(const uint32_t *seeds, int n_seeds, int64_t n, int32_t *tables, void *scratch,
                               int64_t scratch_bytes, int64_t *rounds, xrs_stream_t stream) {
    int rc = table_args(n_seeds, n);
    if (rc) return rc;
    XRS_REQUIRE(seeds != nullptr, "NULL seed list");
    XRS_REQUIRE(tables != nullptr, "NULL tables");
    const TableLayout L(n_seeds, n);
    XRS_TRY(check_scratch(scratch, scratch_bytes, L.total, "xrs_perm_tables_scratch_bytes"));
    cudaStream_t s = (cudaStream_t)stream;
    char *sc = (char *)scratch;
    TableCtl *ctl = (TableCtl *)sc;
    uint32_t *mt = (uint32_t *)(sc + L.mt), *words = (uint32_t *)(sc + L.words), *step = (uint32_t *)(sc + L.step);
    int32_t *J = (int32_t *)(sc + L.J);
    unsigned long long *R = (unsigned long long *)(sc + L.R);
    int32_t *lists[2] = {(int32_t *)(sc + L.list0), (int32_t *)(sc + L.list1)};
    Seeds sd{};
    uint32_t first[kMaxSeeds];
    for (int k = 0; k < n_seeds; ++k) {
        sd.v[k] = seeds[k];
        first[k] = (uint32_t)(n - 1);
    }
    XRS_CUDA(cudaMemcpyAsync(step, first, 4 * n_seeds, cudaMemcpyHostToDevice, s));
    // the draws: chunks of the word streams until every seed has resolved step 1
    for (int chunk = 0;; ++chunk) {
        nz_gen_kernel<<<n_seeds, kGenThreads, 0, s>>>(sd, mt, words, chunk, step);
        XRS_CUDA(cudaGetLastError());
        nz_resolve_kernel<<<n_seeds, 32, 0, s>>>(words, step, J, n);
        XRS_CUDA(cudaGetLastError());
        if (chunk + 1 < kFirstChunks) continue;
        uint32_t left[kMaxSeeds];
        XRS_CUDA(cudaMemcpyAsync(left, step, 4 * n_seeds, cudaMemcpyDeviceToHost, s));
        XRS_CUDA(cudaStreamSynchronize(s));
        if (std::all_of(left, left + n_seeds, [](uint32_t v) { return v == 0; })) break;
        if (chunk + 1 >= kMaxChunks) {
            set_error("xrs_perm_tables: %lld words did not resolve the draws (internal error)",
                      (long long)(kMaxChunks * kChunk));
            return XRS_ECUDA;
        }
    }
    // the swaps: every round commits at least the largest pending step, so n rounds always suffice
    const int64_t total = (int64_t)n_seeds * n;
    XRS_CUDA(cudaMemsetAsync(R, 0, total * 8, s));
    XRS_CUDA(cudaMemsetAsync(ctl, 0, sizeof(TableCtl), s));
    nz_shuffle_init_kernel<<<(unsigned)stride_grid(total), 256, 0, s>>>(tables, lists[0], n_seeds, n);
    XRS_CUDA(cudaGetLastError());
    const int pending = (int)(total - n_seeds);
    XRS_CUDA(cudaMemcpyAsync(&ctl->count[0], &pending, 4, cudaMemcpyHostToDevice, s));
    const unsigned grid = (unsigned)stride_grid(pending);
    int64_t round = 0, used = 0;
    for (;;) {
        for (int j = 0; j < kBatch; ++j) {
            const uint32_t r = (uint32_t)(round + j + 1);
            const int32_t *in = lists[(round + j) & 1];
            nz_reserve_kernel<<<grid, 256, 0, s>>>(in, &ctl->count[j], J, R, n, r);
            XRS_CUDA(cudaGetLastError());
            nz_commit_kernel<<<grid, 256, 0, s>>>(in, &ctl->count[j], lists[(round + j + 1) & 1], &ctl->count[j + 1],
                                                  J, R, tables, n, r);
            XRS_CUDA(cudaGetLastError());
        }
        TableCtl h;
        XRS_CUDA(cudaMemcpyAsync(&h, ctl, sizeof(TableCtl), cudaMemcpyDeviceToHost, s));
        XRS_CUDA(cudaStreamSynchronize(s));
        for (int j = 0; j < kBatch; ++j) used += h.count[j] > 0;
        round += kBatch;
        if (h.count[kBatch] == 0) break;
        if (round > n) {
            set_error("xrs_perm_tables: the shuffle did not finish within %lld rounds (internal error)", (long long)n);
            return XRS_ECUDA;
        }
        XRS_CUDA(cudaMemsetAsync(&ctl->count[0], 0, sizeof(int) * kBatch, s));
        XRS_CUDA(cudaMemcpyAsync(&ctl->count[0], &h.count[kBatch], 4, cudaMemcpyHostToDevice, s));
        XRS_CUDA(cudaMemsetAsync(&ctl->count[kBatch], 0, sizeof(int), s));
    }
    if (rounds) *rounds = used;
    return XRS_OK;
}

extern "C" int xrs_noise_scratch_bytes(int64_t H, int64_t W, int terrain, int64_t *bytes) {
    XRS_REQUIRE(bytes != nullptr, "NULL pointer");
    const int rc = noise_shape(H, W);
    if (rc) return rc;
    *bytes = NoiseLayout(H, W, terrain ? kTerrainOctaves : 1).total;
    return XRS_OK;
}

extern "C" int xrs_noise(const void *in, int dtype, int64_t in_pitch, int64_t H, int64_t W, const int32_t *tables,
                         const float *xs, const float *ys, int terrain, double zfactor, void *out, int64_t out_pitch,
                         int32_t *index_stats, void *scratch, int64_t scratch_bytes, xrs_stream_t stream) {
    int rc = noise_shape(H, W);
    if (rc) return rc;
    XRS_REQUIRE(dtype == XRS_F32 || dtype == XRS_F64, "the noise functions take float32 or float64 cells");
    if (terrain) XRS_TRY(check_cells_arg(in, dtype, kRasterCells, in_pitch, W));
    XRS_REQUIRE(tables != nullptr && xs != nullptr && ys != nullptr, "NULL tables or coordinates");
    XRS_REQUIRE(out != nullptr, "NULL output");
    XRS_TRY(check_out_pitch(out_pitch, cell_size(dtype), W));
    XRS_REQUIRE(index_stats != nullptr, "NULL index_stats");
    const NoiseLayout L(H, W, terrain ? kTerrainOctaves : 1);
    XRS_TRY(check_scratch(scratch, scratch_bytes, L.total, "xrs_noise_scratch_bytes"));
    cudaStream_t s = (cudaStream_t)stream;
    char *sc = (char *)scratch;
    if (dtype == XRS_F32) {
        const float *i = (const float *)in;
        float *o = (float *)out;
        return terrain ? run_noise<float, true>(i, in_pitch / 4, H, W, tables, xs, ys, zfactor, o, out_pitch / 4,
                                                index_stats, sc, L, s)
                       : run_noise<float, false>(i, in_pitch / 4, H, W, tables, xs, ys, zfactor, o, out_pitch / 4,
                                                 index_stats, sc, L, s);
    }
    const double *i = (const double *)in;
    double *o = (double *)out;
    return terrain ? run_noise<double, true>(i, in_pitch / 8, H, W, tables, xs, ys, zfactor, o, out_pitch / 8,
                                             index_stats, sc, L, s)
                   : run_noise<double, false>(i, in_pitch / 8, H, W, tables, xs, ys, zfactor, o, out_pitch / 8,
                                              index_stats, sc, L, s);
}

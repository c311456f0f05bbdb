// box_stream.cu -- convolve_2d with a kernel whose taps are all the same weight w
// (np.ones((k, k)) / k**2: the mean filter of the reference's docs and of benchmarks/; also any
// rectangular kh x kw): out = w * (sum of the window), reference convolution.py:285-313.
//
// A separable RUNNING box on a CTA-wide TMA pipeline: O(1) work per cell for every k.
//   * vertical: every lane keeps the running column sums V of its 4 columns over the last kh rows in
//     float64 registers; per batch of 4 rows:  V_i = V_{i-1} - (row leaving) + (row entering);
//   * horizontal: LANE SUMS.  A lane forms the inclusive prefix `pre` and suffix `suf` of its own 4 column
//     sums and its total; the window of column 4 l + j then is
//         suf[.] of the lane its left end falls in + pre[.] of the lane its right end falls in
//         + the totals of the whole lanes in between,
//     every operand at a compile-time lane distance (RX is a template parameter): 4 (k = 5) ... 11
//     (k = 25) float64 shuffles per lane-row.  The first generation of this kernel ran a 5-step float64
//     prefix scan along the warp and took prefix differences (13 shuffles, a ~600-cycle dependent chain:
//     scripts/tune/box_stream_scan_first_generation.cu.txt).  A NaN that
//     lives in one lane's sums reaches exactly the windows that contain that lane's columns, so the
//     columns beyond the raster's left / right edge (NaN from the TMA unit) need no masking: edge tiles
//     run the fast path and their border windows come out NaN like the reference's;
//   * TWO STREAMS per stage: the 4 rows that enter the window and the 4 rows that leave it (re-read
//     through L2: they were fetched kh rows earlier by the same CTA) arrive as ONE stage with one full /
//     one empty mbarrier -- the ring does not hold the window, so k = 25 gets the same prefetch depth as
//     k = 5, and a consumer warp waits and arrives once per 4 rows;
//   * each warp emits the 128 - 2 * pad(rx) columns whose windows it sees completely; neighbouring warps'
//     input strips overlap in shared memory (free), neighbouring tiles overlap by 2 * pad(rx) columns (L2);
//   * 7 consumer warps + 1 producer warp = 256 threads: 128 registers per thread at two CTAs per SM (no
//     spills in the fast path; 8 + 1 warps are capped at 96 registers: 0.79 instead of 0.87 at k = 9);
//   * row segments are chosen so that no CTA runs one task more than the others (pick_seg_rows).
// H100 SXM (400 W limit), 32768^2 (bench.py `ops`): k = 9 / 25: 286 / 227 Gcells/s = 0.68 / 0.54 of the 3.35 TB/s
// data-sheet HBM bandwidth; outputs bit-identical to the first generation.
// Numerics.  The reference accumulates fma(w, v, acc) tap by tap in float64; here the window sum is
// formed in float64 (sums of float32 cells: rounding ~1e-16 of the window's magnitude) and scaled
// once -- far inside the 1e-5 bar of the float32 result.  Running sums are only trustworthy while
// every cell that entered them is "ordinary": a cell far larger than the data around it (a 1e20
// fill value in a DEM: its float64 ulp is 16384) rounds away the low bits of every other cell of its
// column while it is in V, and subtracting it later does not bring them back, so every later window of
// that column would be wrong.  A cell is therefore EXCEPTIONAL when it is NaN, infinite or at least
// 2^15 x the median |x| of a fixed 128-cell sample of the raster (bs_threshold: one cut-off per launch;
// 2^100 when the sample holds no finite nonzero cell).  Exceptional cells are kept OUT of V and counted
// instead (two 16-bit running counts per column, same lane-sum machinery): a window holding a NaN is NaN
// like the reference's; a window holding an infinite / exceptional cell is recomputed tap by tap in the
// reference's order from global memory; all other windows never saw the bad cell.  Batches without any
// such cell -- one warp vote per 4 rows -- skip the masking and the counts entirely.
#include "stencil3.cuh"

namespace xrs {

constexpr int kBsWarps = 7;      // consumer warps per CTA (+ 1 producer warp)
constexpr int kBsMaxK = 25;      // window rows / columns served
constexpr float kBsHuge = 1.2676506e30f;  // 2^100: the cut-off when the sample holds no finite nonzero cell
constexpr float kBsScale = 32768.f;       // 2^15: cells at or above kBsScale x the sample median are exceptional
constexpr int kB2Rows = 4;       // rows per stage half (entering / leaving)
constexpr int kBoxNotTaken = -12345;

// The launch's cut-off between ordinary cells (summed into V) and exceptional ones (kept out of V, their windows
// recomputed tap by tap): 2^15 x the median |x| of the finite nonzero cells among 128 fixed sample cells
// (sample s = 4 lane + j at row (2 s + 1) H / 256, column (2 ((79 s) mod 128) + 1) W / 256).  Every warp of
// every CTA computes the same value.  A median ignores a few planted sentinels, and a cut-off relative to the
// data keeps any ordinary cell from rounding away more than ~2^-38 of the data's magnitude from a column sum
// (DESIGN section 4.2).  Mirrored by `_box_threshold` in tests/test_kernel_algebra.py.
__device__ __noinline__ float bs_threshold(const float *__restrict__ in, int64_t pitch_elems, int64_t H, int64_t W) {
    const int lane = threadIdx.x & 31;
    float a[4];
    bool ok[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int s = 4 * lane + j;
        const int64_t y = (2 * s + 1) * H / 256, x = (2 * ((79 * s) & 127) + 1) * W / 256;
        a[j] = fabsf(in[y * pitch_elems + x]);
        ok[j] = a[j] > 0.f && a[j] < __int_as_float(0x7f800000);   // NaN fails both
    }
    int rank[4] = {0, 0, 0, 0}, n = 0;
    for (int src = 0; src < 32; ++src) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float b = __shfl_sync(0xffffffffu, a[k], src);
            const bool okb = __shfl_sync(0xffffffffu, ok[k], src);
            n += okb;
#pragma unroll
            for (int j = 0; j < 4; ++j)   // order by (value, sample index): every rank 0 .. n - 1 is held once
                rank[j] += okb && (b < a[j] || (b == a[j] && 4 * src + k < 4 * lane + j));
        }
    }
    unsigned med = 0u;
#pragma unroll
    for (int j = 0; j < 4; ++j)
        if (ok[j] && rank[j] == n / 2) med = __float_as_uint(a[j]);
    med = __reduce_max_sync(0xffffffffu, med);
    return n ? __uint_as_float(med) * kBsScale : kBsHuge;
}

__device__ __noinline__ float bs_direct(const float *__restrict__ in, int64_t pitch_elems, int64_t H, int64_t W,
                                        int64_t y, int64_t x, int kh, int kw, double w) {
    // the reference's tap-order float64 accumulation (convolution.py:303-308); only called for cells
    // off the NaN ring, so every tap is inside the raster
    double acc = 0.0;
    const float *p = in + (y - kh / 2) * pitch_elems + (x - kw / 2);
    for (int ky = 0; ky < kh; ++ky)
        for (int kx = 0; kx < kw; ++kx) acc = fma(w, (double)p[ky * pitch_elems + kx], acc);
    return (float)acc;
}

// focal.apply's mean over an all-ones window (focal.py:268-270 `_calc_mean` = np.nanmean of the window
// scratch, focal.py:305-326): NaN cells and cells beyond the raster are skipped, infinite cells take part
__device__ __noinline__ float bs_direct_nanmean(const float *__restrict__ in, int64_t pitch_elems, int64_t H, int64_t W,
                                                int64_t y, int64_t x, int kh, int kw) {
    double c = 0.0;
    int cnt = 0;
    for (int ky = 0; ky < kh; ++ky) {
        const int64_t yy = y - kh / 2 + ky;
        if (yy < 0 || yy >= H) continue;
        for (int kx = 0; kx < kw; ++kx) {
            const int64_t xx = x - kw / 2 + kx;
            if (xx < 0 || xx >= W) continue;
            const float v = in[yy * pitch_elems + xx];
            if (v == v) { c += (double)v; ++cnt; }
        }
    }
    return (float)(c / (double)cnt);   // an empty window is 0 / 0 = NaN, like np.nanmean
}
// c / n for an integer n with inv = 1 / n correctly rounded: quotient, exact remainder, one correction
// (the float64 quotient numpy forms; checked against rationals in tests/test_kernel_algebra.py)
__device__ __forceinline__ double bs_div_n(double c, double n, double inv) {
    const double q = c * inv;
    return fma(fma(-q, n, c), inv, q);
}

template <int RX, int NW> struct B2Shape {
    static constexpr int kPad = (RX + 3) / 4 * 4;               // columns a warp cannot emit on each side
    static constexpr int kOutW = kStripW - 2 * kPad;            // columns a warp emits
    static constexpr int kTileOutW = NW * kOutW;
    static constexpr int kTileInW = kTileOutW + 2 * kPad;
    static constexpr int kNBox = (kTileInW + 255) / 256;
    static constexpr int kBoxW = ((kTileInW + kNBox - 1) / kNBox + 31) / 32 * 32;   // cells: 128-byte multiples
    static constexpr int kBoxCells = kB2Rows * kBoxW;           // one TMA box: 4 rows x kBoxW cells
    static constexpr int kHalfCells = kNBox * kBoxCells;        // the entering (or leaving) rows of a stage
    static constexpr uint32_t kHalfBytes = kHalfCells * 4;
    static_assert(kBoxW <= 256 && kBoxW % 32 == 0 && kNBox * kBoxW >= kTileInW, "TMA box geometry");
};

struct B2Geom {
    int64_t H, W;
    int kh, ry;
    int n_tiles, n_segs, seg_rows;
    int stages;
    double w;        // MODE 0: the taps' common weight; MODE 1: 1 / (kh * kw)
    double n_cells;  // kh * kw
};

// max(|a|, |b|, |c|), NaN if any operand is NaN (two FMNMX.NAN with |.| operand modifiers)
__device__ __forceinline__ float bs_amax3(float a, float b, float c) {
    return max_nan(max_nan(fabsf(a), fabsf(b)), fabsf(c));
}
__device__ __forceinline__ float bs_amax4(const float (&v)[4]) {
    return bs_amax3(bs_amax3(v[0], v[1], v[2]), v[3], v[3]);
}

// the value lane (l + D) holds; lanes past the warp's ends get their own (they sit in the pad)
template <int D, typename T> __device__ __forceinline__ T bs_from(T x) {
    if constexpr (D == 0) return x;
    else if constexpr (sizeof(T) == 8) {
        // the two halves shuffled as plain 32-bit values: ptxas pairs the results with fewer register moves
        // than through the 64-bit overload (338 instead of 359 instructions per 4-row batch at k = 9)
        int lo = __double2loint(x), hi = __double2hiint(x);
        if constexpr (D > 0) { lo = __shfl_down_sync(0xffffffffu, lo, D); hi = __shfl_down_sync(0xffffffffu, hi, D); }
        else { lo = __shfl_up_sync(0xffffffffu, lo, -D); hi = __shfl_up_sync(0xffffffffu, hi, -D); }
        return __hiloint2double(hi, lo);
    }
    else if constexpr (D > 0) return __shfl_down_sync(0xffffffffu, x, D);
    else return __shfl_up_sync(0xffffffffu, x, -D);
}

// window sum of column 4 l + J (radius RX) from the lane-local prefix / suffix sums, the lane total,
// `core` = the totals of lanes l-q+1 .. l+q-1, `tl` / `tr` = the totals of lanes l-q / l+q  (q = RX / 4)
template <int RX, int J, typename T>
__device__ __forceinline__ T bs_cell(const T (&pre)[4], const T (&suf)[4], T tot, T core, T tl, T tr) {
    constexpr int q = RX / 4, m = RX % 4;
    constexpr int a = J - m, b = J + m;          // window = [4 (l - q) + a, 4 (l + q) + b]
    if constexpr (q == 0 && a >= 0 && b <= 3) {  // inside the lane (RX = 1 only)
        static_assert(a == 0 || b == 3, "in-lane window");
        if constexpr (a == 0) return pre[b]; else return suf[a];
    } else {
        constexpr int dl = -q - (a < 0 ? 1 : 0), ia = (a + 4) & 3;
        constexpr int dh = q + (b >= 4 ? 1 : 0), ib = b & 3;
        const T ends = bs_from<dl>(suf[ia]) + bs_from<dh>(pre[ib]);
        if constexpr (q == 0) {
            if constexpr (a < 0 && b >= 4) return ends + tot; else return ends;
        } else {
            T full = core;
            if constexpr (a < 0) full = full + tl;
            if constexpr (b >= 4) full = full + tr;
            return ends + full;
        }
    }
}

// win[i][j] = sum of v[i] over columns 4 l + j - RX .. 4 l + j + RX, for R independent rows (their
// shuffle / add chains interleave)
template <int RX, int R, typename T>
__device__ __forceinline__ void bs_lanesum(const T (&v)[R][4], T (&win)[R][4]) {
    static_assert(RX >= 1 && RX <= 12, "window radius");
    constexpr int q = RX / 4, m = RX % 4;
#pragma unroll
    for (int i = 0; i < R; ++i) {
        T pre[4], suf[4];
        pre[0] = v[i][0];
        pre[1] = pre[0] + v[i][1];
        pre[2] = pre[1] + v[i][2];
        pre[3] = pre[2] + v[i][3];
        suf[3] = v[i][3];
        suf[2] = v[i][2] + suf[3];
        suf[1] = v[i][1] + suf[2];
        suf[0] = pre[3];
        const T tot = pre[3];
        T core = tot, tl = T(0), tr = T(0);
        if constexpr (q == 2) core = (bs_from<-1>(tot) + tot) + bs_from<1>(tot);
        if constexpr (q == 3) {
            const T pair = tot + bs_from<1>(tot);                       // lanes l, l + 1
            core = (bs_from<-2>(pair) + pair) + bs_from<2>(tot);        // lanes l - 2 .. l + 2
        }
        if constexpr (q >= 1 && m > 0) {
            tl = bs_from<-q>(tot);
            tr = bs_from<q>(tot);
        }
        win[i][0] = bs_cell<RX, 0, T>(pre, suf, tot, core, tl, tr);
        win[i][1] = bs_cell<RX, 1, T>(pre, suf, tot, core, tl, tr);
        win[i][2] = bs_cell<RX, 2, T>(pre, suf, tot, core, tl, tr);
        win[i][3] = bs_cell<RX, 3, T>(pre, suf, tot, core, tl, tr);
    }
}

__device__ __forceinline__ uint32_t bs_bits(int n) { return n >= 32 ? 0xffffffffu : ((1u << n) - 1u); }

// MODE 0: convolve_2d (a NaN anywhere in the window makes the result NaN; raster-edge windows are NaN).
// MODE 1: focal.apply mean over an all-ones window (NaN and out-of-raster cells are skipped).
template <int RX, int NW, int MODE>
__global__ void __launch_bounds__((NW + 1) * 32, 2)
box_stream2_kernel(const __grid_constant__ CUtensorMap tmap, const float *__restrict__ in, int64_t in_pitch_elems,
                   float *__restrict__ out, int64_t out_pitch_elems, const B2Geom g) {
    using S = B2Shape<RX, NW>;
    constexpr int kw = 2 * RX + 1;
    constexpr int kStageCells = 2 * S::kHalfCells;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    float *ring = reinterpret_cast<float *>(smem_raw);
    uint64_t *full = reinterpret_cast<uint64_t *>(smem_raw + (size_t)g.stages * kStageCells * sizeof(float));
    uint64_t *empty = full + g.stages;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmap);
        for (int s = 0; s < g.stages; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], NW);
        }
        mbar_fence_init();
    }
    __syncthreads();

    const int64_t n_tasks = (int64_t)g.n_tiles * g.n_segs;
    const int kh = g.kh, ry = g.ry;

    if (warp == NW) {
        // ---- producer: per task the batches of 4 entering rows e0 .. e0 + 3 (row e = raster row
        // y0 - ry + e) and, once rows leave the window, the 4 rows e0 - (kh - 1) .. that leave with them
        if (lane == 0) {
            int stage = 0;
            uint32_t lap = 0;
            for (int64_t task = blockIdx.x; task < n_tasks; task += gridDim.x) {
                const int seg = (int)(task / g.n_tiles), tile = (int)(task % g.n_tiles);
                const int64_t y0 = (int64_t)seg * g.seg_rows, y1 = min(y0 + (int64_t)g.seg_rows, g.H);
                const int bx = tile * S::kTileOutW - S::kPad;
                const int ytop = (int)y0 - ry;
                const int n_in = (int)(y1 - y0) + kh - 1;
                for (int e0 = 0; e0 < n_in; e0 += kB2Rows) {
                    mbar_wait(&empty[stage], lap ^ 1u);  // a fresh barrier passes the first lap
                    const bool leaving = e0 + kB2Rows - 1 >= kh - 1;
                    mbar_arrive_expect_tx(&full[stage], leaving ? 2u * S::kHalfBytes : S::kHalfBytes);
                    float *dst = ring + (size_t)stage * kStageCells;
#pragma unroll
                    for (int b = 0; b < S::kNBox; ++b)
                        tma_load_2d(dst + b * S::kBoxCells, &tmap, &full[stage], bx + b * S::kBoxW, ytop + e0);
                    if (leaving) {
#pragma unroll
                        for (int b = 0; b < S::kNBox; ++b)
                            tma_load_2d(dst + S::kHalfCells + b * S::kBoxCells, &tmap, &full[stage], bx + b * S::kBoxW,
                                        ytop + e0 - (kh - 1));
                    }
                    if (++stage == g.stages) { stage = 0; lap ^= 1u; }
                }
            }
        }
        return;
    }

    // ---- consumers
    const int col = warp * S::kOutW + 4 * lane;                         // first of the lane's columns in the tile row
    const int off = (col / S::kBoxW) * S::kBoxCells + (col % S::kBoxW);  // + i * kBoxW for row i of the half
    const bool emits = (4 * lane >= S::kPad) && (4 * lane < kStripW - S::kPad);
    const uint32_t win_mask = bs_bits(kh - 1);   // the rows in the window before a row is added
    const float thr = bs_threshold(in, in_pitch_elems, g.H, g.W);
    int stage = 0;
    uint32_t lap = 0;
    for (int64_t task = blockIdx.x; task < n_tasks; task += gridDim.x) {
        const int seg = (int)(task / g.n_tiles), tile = (int)(task % g.n_tiles);
        const int64_t y0 = (int64_t)seg * g.seg_rows, y1 = min(y0 + (int64_t)g.seg_rows, g.H);
        const int64_t x = (int64_t)tile * S::kTileOutW - S::kPad + col;  // raster column of the lane's first cell
        const bool in_raster = x >= 0 && x < g.W;                          // W % 4 == 0: all four cells in or out
        const bool store_ok = emits && in_raster;
        // Out-of-raster columns (NaN from the TMA unit) never vote a row "dirty".  MODE 0: they may poison
        // their own lane's sums -- exactly the windows that contain them must be NaN.  MODE 1 skips them: the
        // lane's cells are read as 0, and a window that reaches beyond the raster's left / right edge divides
        // by the number of columns it really has (ncv) -- edge tiles stay on the fast path in both modes.
        const bool watch = in_raster;
        int ncv[4] = {kw, kw, kw, kw};
        bool edge_warp = false;
        if constexpr (MODE == 1) {
            bool edge_lane = false;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int64_t xc = x + j;
                const int64_t lo = xc - RX < 0 ? 0 : xc - RX, hi = xc + RX > g.W - 1 ? g.W - 1 : xc + RX;
                ncv[j] = (int)(hi - lo + 1);
                edge_lane = edge_lane || (ncv[j] != kw);
            }
            edge_warp = __any_sync(0xffffffffu, edge_lane && in_raster);
        }
        float *optr = out + y0 * out_pitch_elems + x;

        double V[4] = {0.0, 0.0, 0.0, 0.0};
        unsigned C[4] = {0u, 0u, 0u, 0u};   // lo 16 bits: NaN cells in the column window, hi 16: infinite / huge
        uint32_t dirty = 0;                  // bit i: the row added i rows ago held a NaN / inf / huge cell (this warp)
        const int n_in = (int)(y1 - y0) + kh - 1;
        for (int e0 = 0; e0 < n_in; e0 += kB2Rows) {
            mbar_wait(&full[stage], lap);
            const float *se = ring + (size_t)stage * kStageCells + off;   // entering rows
            const float *sl = se + S::kHalfCells;                          // leaving rows
            bool done = false;
            if (e0 >= kh - 1 && e0 + kB2Rows <= n_in && (dirty & win_mask) == 0u) {
                // ---- fast path: window complete, 4 rows enter, 4 rows are emitted, 4 rows leave; neither
                // the window nor the entering rows hold a NaN / inf / huge cell inside the raster
                float nv[kB2Rows][4];
#pragma unroll
                for (int i = 0; i < kB2Rows; ++i) {
                    const float4 q = *reinterpret_cast<const float4 *>(se + i * S::kBoxW);
                    nv[i][0] = q.x; nv[i][1] = q.y; nv[i][2] = q.z; nv[i][3] = q.w;
                }
                if constexpr (MODE == 1) {
                    if (edge_warp && !in_raster) {   // only warps at the raster's left / right edge hold such lanes
#pragma unroll
                        for (int i = 0; i < kB2Rows; ++i) { nv[i][0] = 0.f; nv[i][1] = 0.f; nv[i][2] = 0.f; nv[i][3] = 0.f; }
                    }
                }
                const float amax = bs_amax3(bs_amax3(bs_amax4(nv[0]), nv[1][0], nv[1][1]),
                                            bs_amax3(bs_amax4(nv[2]), nv[1][2], nv[1][3]), bs_amax4(nv[3]));
                if (!__any_sync(0xffffffffu, watch && !(amax < thr))) {
                    float ov[kB2Rows][4];
#pragma unroll
                    for (int i = 0; i < kB2Rows; ++i) {
                        const float4 q = *reinterpret_cast<const float4 *>(sl + i * S::kBoxW);
                        ov[i][0] = q.x; ov[i][1] = q.y; ov[i][2] = q.z; ov[i][3] = q.w;
                    }
                    if constexpr (MODE == 1) {
                        if (edge_warp && !in_raster) {
#pragma unroll
                            for (int i = 0; i < kB2Rows; ++i) { ov[i][0] = 0.f; ov[i][1] = 0.f; ov[i][2] = 0.f; ov[i][3] = 0.f; }
                        }
                    }
                    // column sums of output row i: V_i = V_{i-1} - old_{i-1} + new_i
                    double P[kB2Rows][4];
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        double acc = V[j];
#pragma unroll
                        for (int i = 0; i < kB2Rows; ++i) {
                            const double d = (i == 0) ? (double)nv[0][j] : ((double)nv[i][j] - (double)ov[i > 0 ? i - 1 : 0][j]);
                            acc += d;
                            P[i][j] = acc;
                        }
                        V[j] = acc - (double)ov[kB2Rows - 1][j];
                    }
                    double win[kB2Rows][4];
                    bs_lanesum<RX, kB2Rows, double>(P, win);
#pragma unroll
                    for (int i = 0; i < kB2Rows; ++i) {
                        if (store_ok) {
                            if constexpr (MODE == 0)
                                __stcs(reinterpret_cast<float4 *>(optr),
                                       make_float4((float)fma(g.w, win[i][0], 0.0), (float)fma(g.w, win[i][1], 0.0),
                                                   (float)fma(g.w, win[i][2], 0.0), (float)fma(g.w, win[i][3], 0.0)));
                            else if (!edge_warp)
                                __stcs(reinterpret_cast<float4 *>(optr),
                                       make_float4((float)bs_div_n(win[i][0], g.n_cells, g.w), (float)bs_div_n(win[i][1], g.n_cells, g.w),
                                                   (float)bs_div_n(win[i][2], g.n_cells, g.w), (float)bs_div_n(win[i][3], g.n_cells, g.w)));
                            else
                                __stcs(reinterpret_cast<float4 *>(optr),
                                       make_float4((float)(win[i][0] / (double)(kh * ncv[0])), (float)(win[i][1] / (double)(kh * ncv[1])),
                                                   (float)(win[i][2] / (double)(kh * ncv[2])), (float)(win[i][3] / (double)(kh * ncv[3]))));
                        }
                        optr += out_pitch_elems;
                    }
                    dirty <<= kB2Rows;
                    done = true;
                }
            }
            if (!done) {
                // ---- row by row: lead-in rows (nothing to emit yet), the last rows of a task, and windows
                // or entering rows with NaN / inf / huge cells (kept out of V, counted in C)
                for (int i = 0; i < kB2Rows; ++i) {
                    const int e = e0 + i;
                    if (e >= n_in) break;
                    const float4 q = *reinterpret_cast<const float4 *>(se + i * S::kBoxW);
                    const bool zero_lane = MODE == 1 && !in_raster;
                    const float v[4] = {zero_lane ? 0.f : q.x, zero_lane ? 0.f : q.y, zero_lane ? 0.f : q.z, zero_lane ? 0.f : q.w};
                    const bool row_dirty = __any_sync(0xffffffffu, watch && !(bs_amax4(v) < thr));
                    dirty = (dirty << 1) | (row_dirty ? 1u : 0u);
                    if (!row_dirty) {
#pragma unroll
                        for (int j = 0; j < 4; ++j) V[j] += (double)v[j];
                    } else {
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const bool isnan_ = v[j] != v[j];
                            const bool big = !isnan_ && !(fabsf(v[j]) < thr);
                            V[j] += (isnan_ || big) ? 0.0 : (double)v[j];
                            C[j] += isnan_ ? 1u : (big ? 0x10000u : 0u);
                        }
                    }
                    if (e < kh - 1) continue;   // window not complete yet

                    // emit output row y = y0 + e - (kh - 1)
                    const bool win_dirty = (dirty & bs_bits(kh)) != 0u;
                    double P1[1][4] = {{V[0], V[1], V[2], V[3]}}, w1[1][4];
                    bs_lanesum<RX, 1, double>(P1, w1);
                    float res[4];
#pragma unroll
                    for (int j = 0; j < 4; ++j)
                        res[j] = MODE == 0 ? (float)fma(g.w, w1[0][j], 0.0)    // + 0.0: an all-zero window is +0 like the reference's
                                 : (edge_warp ? (float)(w1[0][j] / (double)(kh * ncv[j])) : (float)bs_div_n(w1[0][j], g.n_cells, g.w));
                    if (win_dirty) {   // warp-uniform
                        unsigned C1[1][4] = {{C[0], C[1], C[2], C[3]}}, wc[1][4];
                        bs_lanesum<RX, 1, unsigned>(C1, wc);
                        const int64_t y = y0 + e - (kh - 1);
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            if constexpr (MODE == 0) {
                                if (wc[0][j] & 0xffffu) res[j] = nan_of<float>();
                                else if (wc[0][j] >> 16) {
                                    if (store_ok) res[j] = bs_direct(in, in_pitch_elems, g.H, g.W, y, x + j, kh, kw, g.w);
                                }
                            } else {
                                if (wc[0][j] >> 16) {          // infinite / huge cells take part: the reference's order
                                    if (store_ok) res[j] = bs_direct_nanmean(in, in_pitch_elems, g.H, g.W, y, x + j, kh, kw);
                                } else if (wc[0][j] & 0xffffu) {
                                    res[j] = (float)(w1[0][j] / (double)(kh * ncv[j] - (int)(wc[0][j] & 0xffffu)));   // all skipped: 0 / 0 = NaN
                                }
                            }
                        }
                    }
                    if (store_ok) __stcs(reinterpret_cast<float4 *>(optr), make_float4(res[0], res[1], res[2], res[3]));
                    optr += out_pitch_elems;

                    // retire input row e - (kh - 1), the oldest row of the window
                    const float4 qo = *reinterpret_cast<const float4 *>(sl + i * S::kBoxW);
                    const float vo[4] = {zero_lane ? 0.f : qo.x, zero_lane ? 0.f : qo.y, zero_lane ? 0.f : qo.z, zero_lane ? 0.f : qo.w};
                    const bool old_dirty = (dirty >> (kh - 1)) & 1u;
                    if (!old_dirty) {
#pragma unroll
                        for (int j = 0; j < 4; ++j) V[j] -= (double)vo[j];
                    } else {
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const bool isnan_ = vo[j] != vo[j];
                            const bool big = !isnan_ && !(fabsf(vo[j]) < thr);
                            V[j] -= (isnan_ || big) ? 0.0 : (double)vo[j];
                            C[j] -= isnan_ ? 1u : (big ? 0x10000u : 0u);
                        }
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[stage]);
            if (++stage == g.stages) { stage = 0; lap ^= 1u; }
        }
    }
}

template <int RX, int NW, int MODE>
static int launch_box_stream2(const float *in, int64_t in_pitch, float *out, int64_t out_pitch, int64_t H, int64_t W,
                              int kh, double w, cudaStream_t s) {
    using S = B2Shape<RX, NW>;
    CUtensorMap tmap;
    if (!make_tensor_map_2d(&tmap, in, in_pitch, H, W, XRS_F32, S::kBoxW, kB2Rows)) return kBoxNotTaken;
    B2Geom g;
    g.H = H; g.W = W; g.kh = kh; g.ry = kh / 2; g.w = w;
    g.n_cells = (double)(kh * (2 * RX + 1));
    g.n_tiles = (int)((W + S::kTileOutW - 1) / S::kTileOutW);
    int stages = RX <= 2 ? 3 : 4, max_ctas = 2, want = 4;   // swept with scripts/tune/box_zonal_sweep.py
    if (const char *e = getenv("XRS_BOX_STAGES")) stages = atoi(e);
    if (const char *e = getenv("XRS_BOX_CTAS")) max_ctas = atoi(e);
    if (const char *e = getenv("XRS_BOX_WAVES")) want = atoi(e);
    if (max_ctas < 1) max_ctas = 1;
    if (want < 1) want = 1;
    const size_t stage_bytes = (size_t)2 * S::kHalfBytes;
    const size_t cap = (kSmemPerSm - (size_t)max_ctas * kSmemReservedPerCta) / max_ctas - 256;
    if (stages < 2) stages = 2;
    while (stages > 2 && (size_t)stages * stage_bytes + (size_t)2 * stages * sizeof(uint64_t) > cap) --stages;
    g.stages = stages;
    const size_t smem = (size_t)stages * stage_bytes + (size_t)2 * stages * sizeof(uint64_t);
    auto kern = box_stream2_kernel<RX, NW, MODE>;
    int64_t resident;
    if (const int rc = resident_ctas(kern, (NW + 1) * 32, smem, max_ctas, &resident)) return rc;
    // segments: tall enough that the kh - 1 lead-in rows stay a small overhead, (rows + kh - 1) a
    // multiple of 4 so that only the raster's last segment ends in a partial batch
    const int64_t seg_rows = pick_seg_rows(H, g.n_tiles, resident, 12 * (int64_t)kh, kh - 1, kB2Rows, want);
    g.seg_rows = (int)seg_rows;
    g.n_segs = (int)((H + seg_rows - 1) / seg_rows);
    const int64_t n_tasks = (int64_t)g.n_tiles * g.n_segs;
    return launch(kern, resident < n_tasks ? resident : n_tasks, (NW + 1) * 32, smem, s, kRunningBox, tmap, in,
                  in_pitch / 4, out, out_pitch / 4, g);
}

// true when the streaming box kernel took the job (*rc = its status)
bool try_box_stream(const float *in, int64_t in_pitch, float *out, int64_t out_pitch, int64_t H, int64_t W,
                    const double *kernel, int kh, int kw, cudaStream_t s, int *rc) {
    if (kh > kBsMaxK || kw > kBsMaxK || kh < 1 || kw < 3 || (kw & 1) == 0 || (kh & 1) == 0) return false;
    const double w = kernel[0];
    if (!(fabs(w) <= 1.7976931348623157e308)) return false;
    for (int i = 1; i < kh * kw; ++i)
        if (memcmp(&kernel[i], &w, sizeof(double)) != 0) return false;
    if (W % 4 != 0 || out_pitch % 16 != 0 || (reinterpret_cast<uintptr_t>(out) & 15)) return false;
    if (H >= (1LL << 31) - 64 || W >= (1LL << 31) - 4096) return false;
    int r2 = kBoxNotTaken;
    switch (kw / 2) {
#define XRS_BS(R) case R: r2 = launch_box_stream2<R, kBsWarps, 0>(in, in_pitch, out, out_pitch, H, W, kh, w, s); break;
        XRS_BS(1) XRS_BS(2) XRS_BS(3) XRS_BS(4) XRS_BS(5) XRS_BS(6) XRS_BS(7) XRS_BS(8) XRS_BS(9) XRS_BS(10) XRS_BS(11) XRS_BS(12)
#undef XRS_BS
    }
    if (r2 == kBoxNotTaken) return false;     // TMA cannot describe the raster: the tiled kernels take it
    *rc = r2;
    return true;
}

// focal.apply(mean) over an all-ones kh x kw window (the reference's own focal benchmark, benchmarks/focal.py
// FocalApply): the same running box in NaN-skipping mode.  true when it took the job (*rc = its status)
bool try_box_nanmean(const float *in, int64_t in_pitch, float *out, int64_t out_pitch, int64_t H, int64_t W,
                     int kh, int kw, cudaStream_t s, int *rc) {
    if (kh > kBsMaxK || kw > kBsMaxK || kh < 1 || kw < 3 || (kw & 1) == 0 || (kh & 1) == 0) return false;
    if (W % 4 != 0 || out_pitch % 16 != 0 || (reinterpret_cast<uintptr_t>(out) & 15)) return false;
    if (H >= (1LL << 31) - 64 || W >= (1LL << 31) - 4096) return false;
    const double w = 1.0 / (double)(kh * kw);
    int r2 = kBoxNotTaken;
    switch (kw / 2) {
#define XRS_BS(R) case R: r2 = launch_box_stream2<R, kBsWarps, 1>(in, in_pitch, out, out_pitch, H, W, kh, w, s); break;
        XRS_BS(1) XRS_BS(2) XRS_BS(3) XRS_BS(4) XRS_BS(5) XRS_BS(6) XRS_BS(7) XRS_BS(8) XRS_BS(9) XRS_BS(10) XRS_BS(11) XRS_BS(12)
#undef XRS_BS
    }
    if (r2 == kBoxNotTaken) return false;
    *rc = r2;
    return true;
}

}  // namespace xrs

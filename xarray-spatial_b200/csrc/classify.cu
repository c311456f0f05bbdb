// classify.cu -- the device work behind classify.py (classify.py of the reference, NumPy path):
//   * one per-cell pass for every scheme: the reference's binary-search bin lookup (_cpu_bin) or the
//     membership test of `binary` (_cpu_binary), bins and values in shared memory;
//   * one reduction of the finite cells (optionally only those above a threshold): count, mean, M2, min, max;
//   * a batched radix select: the exact r-th smallest key for many ranks in one set of 8-bit digit passes;
//   * an LSD radix sort of the finite keys, and the gap / pick passes of maximum_breaks over the sorted keys.
// Keys are order-preserving unsigned images of the cell bits, -0.0 folded into +0.0.
#include <math.h>

#include <algorithm>
#include <vector>

#include "common.cuh"

namespace xrs {
namespace {

constexpr int kThreads = 256, kItems = 4, kChunk = kThreads * kItems;
constexpr int kMaxGroups = 128;        // select: target prefixes one histogram launch serves (128 KB of counters)
constexpr int kSortItems = 8, kSortTile = kThreads * kSortItems, kWarps = kThreads / 32;

template <typename T> __device__ __forceinline__ bool finite_cell(T v) {
    if constexpr (std::is_floating_point_v<T>) return isfinite(v);
    else return true;
}

template <typename T> __device__ __forceinline__ uint64_t key_of(T v) {
    if constexpr (std::is_same_v<T, float>) {
        const uint32_t u = v == 0.0f ? 0u : __float_as_uint(v);
        return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    } else if constexpr (std::is_same_v<T, double>) {
        const uint64_t u = v == 0.0 ? 0ull : (uint64_t)__double_as_longlong(v);
        return (u & 0x8000000000000000ull) ? ~u : (u | 0x8000000000000000ull);
    } else if constexpr (std::is_same_v<T, int32_t>) {
        return (uint32_t)v ^ 0x80000000u;
    } else if constexpr (std::is_same_v<T, int64_t>) {
        return (uint64_t)v ^ 0x8000000000000000ull;
    } else if constexpr (std::is_same_v<T, int16_t>) {
        return (uint16_t)v ^ 0x8000u;
    } else {
        static_assert(std::is_same_v<T, uint16_t>, "cell type");
        return v;
    }
}

template <typename T> __device__ __forceinline__ T value_of(uint64_t k) {
    if constexpr (std::is_same_v<T, float>) {
        const uint32_t u = (uint32_t)k;
        return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
    } else if constexpr (std::is_same_v<T, double>) {
        return __longlong_as_double((long long)((k & 0x8000000000000000ull) ? (k & 0x7fffffffffffffffull) : ~k));
    } else if constexpr (std::is_same_v<T, int32_t>) {
        return (int32_t)((uint32_t)k ^ 0x80000000u);
    } else if constexpr (std::is_same_v<T, int64_t>) {
        return (int64_t)(k ^ 0x8000000000000000ull);
    } else if constexpr (std::is_same_v<T, int16_t>) {
        return (int16_t)(uint16_t)((uint32_t)k ^ 0x8000u);
    } else {
        return (uint16_t)k;
    }
}

// a cell from the low bits of `u`, and a cell's bits
template <typename T> __device__ __forceinline__ T from_bits(uint64_t u) {
    if constexpr (std::is_same_v<T, float>) return __uint_as_float((uint32_t)u);
    else if constexpr (std::is_same_v<T, double>) return __longlong_as_double((long long)u);
    else return (T)(std::make_unsigned_t<T>)u;
}
template <typename T> __device__ __forceinline__ uint64_t to_bits(T v) {
    if constexpr (std::is_same_v<T, float>) return __float_as_uint(v);
    else if constexpr (std::is_same_v<T, double>) return (uint64_t)__double_as_longlong(v);
    else return (uint64_t)(std::make_unsigned_t<T>)v;
}

// b - a in the cell type, as np.diff computes it: IEEE for floats, wrapping for integers
template <typename T> __device__ __forceinline__ T diff_of(T b, T a) {
    if constexpr (std::is_floating_point_v<T>) return b - a;
    else {
        using U = std::make_unsigned_t<T>;
        return (T)(U)((U)b - (U)a);
    }
}

// Deals the H x cpr tasks (row, chunk) to the CTAs round robin; one 64-bit division per thread, not per task.
// The bounds are uniform across the CTA, so warp-collective work inside `f` sees every lane.  f(row, chunk).
template <typename F> __device__ __forceinline__ void for_each_task(int64_t H, int64_t cpr, F &&f) {
    if (cpr <= 0 || (int64_t)blockIdx.x >= H * cpr) return;
    int64_t r = (int64_t)blockIdx.x / cpr, k = (int64_t)blockIdx.x - r * cpr;
    const int64_t dr = (int64_t)gridDim.x / cpr, dk = (int64_t)gridDim.x - dr * cpr;
    while (r < H) {
        f(r, k);
        k += dk;
        r += dr;
        if (k >= cpr) {
            k -= cpr;
            ++r;
        }
    }
}

// Visits the cells of an H x W raster in chunks of one row, kChunk columns wide.  f(row, first column of this
// thread: it takes that and the next kItems - 1 columns kThreads apart).
template <typename F> __device__ __forceinline__ void for_each_chunk(int64_t H, int64_t W, F &&f) {
    for_each_task(H, (W + kChunk - 1) / kChunk, [&](int64_t r, int64_t k) { f(r, k * kChunk + threadIdx.x); });
}

template <typename T> __device__ __forceinline__ const T *row_of(const char *base, int64_t pitch, int64_t r) {
    return reinterpret_cast<const T *>(base + r * pitch);
}

// ----------------------------------------------------------------------------- per-cell pass
// classify.py:153-187 `_cpu_bin`, line for line: numba compares the cell and the bin in float64, wraps
// `bins[mid - 1]` at mid = 0, and floors `(end + start) // 2`.  -1: no bin (NaN).
__device__ __forceinline__ int bin_of(double val, const double *bins, int nb) {
    if (!isfinite(val) || nb == 0) return -1;
    if (val <= bins[0]) return 0;
    if (!(val <= bins[nb - 1])) return -1;
    int start = 0, end = nb - 1, mid = (end + start) >> 1;
    while (start <= end) {
        if (bins[mid] < val) start = mid + 1;
        else if (val > bins[mid == 0 ? nb - 1 : mid - 1]) break;
        else end = mid - 1;
        mid = (end + start) >> 1;
    }
    return mid;
}

// _cpu_binary's cell: 1 on a hit, else 0 for a finite cell and NaN for another
template <typename T> __device__ __forceinline__ T member_out(T v, bool hit) {
    if constexpr (std::is_floating_point_v<T>) return hit ? T(1) : (finite_cell(v) ? T(0) : nan_of<T>());
    else return hit ? T(1) : T(0);
}

template <typename T, bool kMember> __device__ __forceinline__ std::conditional_t<kMember, T, float> classify_one(
    T v, const double *bins, const float *newv, int nb) {
    const double x = (double)v;
    if constexpr (kMember) {
        unsigned hit = 0;
        for (int j = 0; j < nb; ++j) hit |= (unsigned)(x == bins[j]);
        return member_out(v, hit != 0);
    } else {
        const int b = bin_of(x, bins, nb);
        return b >= 0 ? newv[b] : nan_of<float>();
    }
}

// kMember false: float32 out, new_values[bin] or NaN.  kMember true (`binary`): out has the cell type, 1 where
// the cell equals one of the nb values (in float64), else 0 for a finite cell and NaN for another.  Each thread
// takes two runs of 16 bytes of cells per row chunk, each one vector load where its address is 16-byte aligned
// and one vector store where the output's address is aligned too.
template <typename T, bool kMember>
__global__ void __launch_bounds__(kThreads) classify_cells_kernel(const char *__restrict__ in, int64_t in_pitch,
                                                                  int64_t H, int64_t W,
                                                                  const double *__restrict__ gbins,
                                                                  const float *__restrict__ gnew, int nb,
                                                                  int in_smem, char *__restrict__ out,
                                                                  int64_t out_pitch) {
    extern __shared__ double smem[];
    const double *bins = gbins;
    const float *newv = gnew;
    if (in_smem) {
        float *sn = reinterpret_cast<float *>(smem + nb);
        for (int i = threadIdx.x; i < nb; i += kThreads) {
            smem[i] = gbins[i];
            if (!kMember) sn[i] = gnew[i];
        }
        __syncthreads();
        bins = smem;
        newv = sn;
    }
    using O = std::conditional_t<kMember, T, float>;
    constexpr int V = 16 / sizeof(T);
    // the cells of one 16-byte load q at row r, column c
    auto vector = [&](const int4 q, int64_t r, int64_t c) {
        const uint32_t w[4] = {(uint32_t)q.x, (uint32_t)q.y, (uint32_t)q.z, (uint32_t)q.w};
        T x[V];
#pragma unroll
        for (int k = 0; k < V; ++k) {
            if constexpr (sizeof(T) == 2) x[k] = from_bits<T>(w[k / 2] >> (16 * (k & 1)));
            else if constexpr (sizeof(T) == 4) x[k] = from_bits<T>(w[k]);
            else x[k] = from_bits<T>((uint64_t)w[2 * k] | ((uint64_t)w[2 * k + 1] << 32));
        }
        uint32_t hits = 0;   // binary: bit k when cell k equals one of the values
        if constexpr (kMember) {
            for (int j = 0; j < nb; ++j) {
                const double b = bins[j];
#pragma unroll
                for (int k = 0; k < V; ++k) hits |= (uint32_t)((double)x[k] == b) << k;
            }
        }
        uint32_t o[V * sizeof(O) / 4] = {};   // the outputs' bits, 32 at a time
#pragma unroll
        for (int k = 0; k < V; ++k) {
            O y;
            if constexpr (kMember) y = member_out(x[k], (hits >> k) & 1u);
            else y = classify_one<T, false>(x[k], bins, newv, nb);
            const uint64_t u = to_bits(y);
            if constexpr (sizeof(O) == 2) o[k / 2] |= (uint32_t)u << (16 * (k & 1));
            else if constexpr (sizeof(O) == 4) o[k] = (uint32_t)u;
            else {
                o[2 * k] = (uint32_t)u;
                o[2 * k + 1] = (uint32_t)(u >> 32);
            }
        }
        char *dst = out + r * out_pitch + c * (int64_t)sizeof(O);
        if (reinterpret_cast<uintptr_t>(dst) % (V * sizeof(O) >= 16 ? 16 : V * sizeof(O)) != 0) {
            // a row of the output not aligned like the input's: one store per cell, from the same bits
#pragma unroll
            for (int k = 0; k < V; ++k) {
                if constexpr (sizeof(O) == 2)
                    __stcs(reinterpret_cast<unsigned short *>(dst) + k, (unsigned short)(o[k / 2] >> (16 * (k & 1))));
                else if constexpr (sizeof(O) == 4)
                    __stcs(reinterpret_cast<unsigned int *>(dst) + k, o[k]);
                else
                    __stcs(reinterpret_cast<unsigned long long *>(dst) + k,
                           (unsigned long long)o[2 * k] | ((unsigned long long)o[2 * k + 1] << 32));
            }
        } else if constexpr (V * sizeof(O) == 8) {
            __stcs(reinterpret_cast<int2 *>(dst), make_int2((int)o[0], (int)o[1]));
        } else {
#pragma unroll
            for (int i = 0; i < (int)(V * sizeof(O) / 16); ++i)
                __stcs(reinterpret_cast<int4 *>(dst) + i,
                       make_int4((int)o[4 * i], (int)o[4 * i + 1], (int)o[4 * i + 2], (int)o[4 * i + 3]));
        }
    };
    auto scalar = [&](int64_t r, int64_t c) {
        const T *src = row_of<T>(in, in_pitch, r);
        O *dst = reinterpret_cast<O *>(out + r * out_pitch);
        for (int k = 0; k < V && c + k < W; ++k)
            __stcs(dst + c + k, classify_one<T, kMember>(__ldcs(src + c + k), bins, newv, nb));
    };
    // two vectors per thread and chunk, both loads issued before either is used
    const int64_t span = 2 * (int64_t)kThreads * V;
    for_each_task(H, (W + span - 1) / span, [&](int64_t r, int64_t chunk) {
        const int64_t c0 = chunk * span + (int64_t)threadIdx.x * V, c1 = c0 + (int64_t)kThreads * V;
        const int4 *src = reinterpret_cast<const int4 *>(row_of<T>(in, in_pitch, r) + c0);
        // a whole vector inside the row, at a 16-byte aligned address (every one of them when the row starts
        // aligned; a row's partial last vector and rows of an unaligned pitch take the scalar path)
        const bool al = reinterpret_cast<uintptr_t>(src) % 16 == 0;
        const bool v0 = al && c0 + V <= W, v1 = al && c1 + V <= W;
        const int4 q0 = v0 ? __ldcs(src) : make_int4(0, 0, 0, 0);
        const int4 q1 = v1 ? __ldcs(src + kThreads) : make_int4(0, 0, 0, 0);
        if (v0) vector(q0, r, c0);
        else scalar(r, c0);
        if (v1) vector(q1, r, c1);
        else scalar(r, c1);
    });
}

// ----------------------------------------------------------------------------- finite moments
struct Moments {
    double n, mean, m2, mn, mx;
};

// Chan et al.'s pairwise update: exact in the counts, stable in M2
__device__ __forceinline__ Moments merge(const Moments &a, const Moments &b) {
    if (a.n == 0.0) return b;
    if (b.n == 0.0) return a;
    Moments m;
    m.n = a.n + b.n;
    const double d = b.mean - a.mean;
    m.mean = a.mean + d * (b.n / m.n);
    m.m2 = a.m2 + b.m2 + d * d * (a.n * (b.n / m.n));
    m.mn = fmin(a.mn, b.mn);
    m.mx = fmax(a.mx, b.mx);
    return m;
}

__device__ __forceinline__ Moments shfl_xor(const Moments &a, int o) {
    return {__shfl_xor_sync(0xffffffffu, a.n, o), __shfl_xor_sync(0xffffffffu, a.mean, o),
            __shfl_xor_sync(0xffffffffu, a.m2, o), __shfl_xor_sync(0xffffffffu, a.mn, o),
            __shfl_xor_sync(0xffffffffu, a.mx, o)};
}

// every lane of the CTA gets the CTA's merge of `m` (fixed order: deterministic)
__device__ __forceinline__ Moments block_merge(Moments m) {
    __shared__ Moments part[kWarps];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = merge(m, shfl_xor(m, o));
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = m;
    __syncthreads();
    Moments r = part[0];
    for (int w = 1; w < kWarps; ++w) r = merge(r, part[w]);
    __syncthreads();
    return r;
}

// Each thread keeps sums shifted by the first cell it counts, so M2 never cancels against the mean's square.
template <typename T>
__global__ void __launch_bounds__(kThreads) moments_kernel(const char *__restrict__ in, int64_t in_pitch, int64_t H,
                                                           int64_t W, double above, Moments *__restrict__ partial) {
    double piv = 0.0, s1 = 0.0, s2 = 0.0, cnt = 0.0, mn = INFINITY, mx = -INFINITY;
    for_each_chunk(H, W, [&](int64_t r, int64_t c0) {
        const T *src = row_of<T>(in, in_pitch, r);
        T v[kItems];
#pragma unroll
        for (int k = 0; k < kItems; ++k) {
            const int64_t c = c0 + k * kThreads;
            v[k] = c < W ? __ldcs(src + c) : T(0);
        }
#pragma unroll
        for (int k = 0; k < kItems; ++k) {
            const double x = (double)v[k];
            if (c0 + k * kThreads < W && finite_cell(v[k]) && x > above) {
                if (cnt == 0.0) piv = x;
                const double d = x - piv;
                s1 += d;
                s2 += d * d;
                cnt += 1.0;
                mn = fmin(mn, x);
                mx = fmax(mx, x);
            }
        }
    });
    Moments m{cnt, 0.0, 0.0, mn, mx};
    if (cnt > 0.0) {
        m.mean = piv + s1 / cnt;
        m.m2 = fmax(s2 - s1 * (s1 / cnt), 0.0);
    }
    m = block_merge(m);
    if (threadIdx.x == 0) partial[blockIdx.x] = m;
}

__global__ void __launch_bounds__(kThreads) moments_finish_kernel(const Moments *__restrict__ partial, int np,
                                                                  double *__restrict__ out) {
    Moments m{0.0, 0.0, 0.0, INFINITY, -INFINITY};
    for (int i = threadIdx.x; i < np; i += kThreads) {
        const Moments &p = partial[i];
        m = merge(m, Moments{p.n, p.mean, p.m2, p.mn, p.mx});
    }
    m = block_merge(m);
    if (threadIdx.x == 0) {
        out[0] = m.n;
        out[1] = m.mean;
        out[2] = m.m2;
        out[3] = m.mn;
        out[4] = m.mx;
    }
}

// ----------------------------------------------------------------------------- key sources
// A source maps (row, col) to a key, or to nothing.  The raster's finite cells:
template <typename T> struct CellKeys {
    const char *base;
    int64_t pitch;
    __device__ __forceinline__ bool key(int64_t r, int64_t c, uint64_t &k) const {
        const T v = __ldcs(row_of<T>(base, pitch, r) + c);
        k = key_of(v);
        return finite_cell(v);
    }
};

// The gaps of np.diff(np.unique(values)) over the sorted keys s (one row): position i > 0 holds the gap
// uv[j] - uv[j - 1] (in the cell type) when s[i] starts a new unique value; the gap's order in np.diff is the
// order of i.
template <typename T, typename K> struct GapKeys {
    const K *s;
    __device__ __forceinline__ bool key(int64_t, int64_t i, uint64_t &k) const {
        if (i == 0) return false;
        const K a = s[i - 1], b = s[i];
        if (a == b) return false;
        k = key_of(diff_of(value_of<T>(b), value_of<T>(a)));
        return true;
    }
};

// The positions of the gaps whose key is `tie`: argsort(kind='stable') orders equal gaps by position.
template <typename T, typename K> struct TiePositions {
    GapKeys<T, K> g;
    uint64_t tie;
    __device__ __forceinline__ bool key(int64_t r, int64_t i, uint64_t &k) const {
        uint64_t gk;
        if (!g.key(r, i, gk) || gk != tie) return false;
        k = (uint64_t)i;
        return true;
    }
};

// ----------------------------------------------------------------------------- batched radix select
// Adds each lane's key to counter `bin` of h (none when bin < 0).  Neighbouring cells of a smooth raster mostly
// share the high digits: a warp whose lanes all hold the same counter adds 32 from one lane instead of
// serialising 32 atomics on one address; other warps add lane by lane.
__device__ __forceinline__ void count_warp(unsigned *h, int bin, unsigned lane) {
    const int first = __shfl_sync(0xffffffffu, bin, 0);
    if (__all_sync(0xffffffffu, bin == first)) {
        if (lane == 0 && first >= 0) atomicAdd(&h[first], 32u);
    } else if (bin >= 0) {
        atomicAdd(&h[bin], 1u);
    }
}

// hist[g * 256 + d] += the keys whose bits above `lo + 8` equal prefix[g] (sorted ascending) and whose digit at
// `lo` is d.
template <typename Src>
__global__ void __launch_bounds__(kThreads) select_hist_kernel(Src src, int64_t H, int64_t W,
                                                               const uint64_t *__restrict__ prefix, int G, int lo,
                                                               unsigned long long *__restrict__ hist) {
    extern __shared__ unsigned sh_hist[];
    __shared__ uint64_t sh_prefix[kMaxGroups];
    for (int i = threadIdx.x; i < G * 256; i += kThreads) sh_hist[i] = 0;
    for (int i = threadIdx.x; i < G; i += kThreads) sh_prefix[i] = prefix[i];
    __syncthreads();
    const int hi = lo + 8;
    const unsigned lane = threadIdx.x & 31;
    for_each_chunk(H, W, [&](int64_t r, int64_t c0) {
#pragma unroll
        for (int k = 0; k < kItems; ++k) {
            const int64_t c = c0 + k * kThreads;
            uint64_t key = 0;
            int bin = -1;
            if (c < W && src.key(r, c, key)) {
                const uint64_t p = hi >= 64 ? 0ull : key >> hi;
                int a = 0, b = G - 1;
                while (a < b) {
                    const int m = (a + b) >> 1;
                    if (sh_prefix[m] < p) a = m + 1;
                    else b = m;
                }
                if (sh_prefix[a] == p) bin = a * 256 + (int)((key >> lo) & 255u);
            }
            count_warp(sh_hist, bin, lane);
        }
    });
    __syncthreads();
    for (int i = threadIdx.x; i < G * 256; i += kThreads)
        if (sh_hist[i]) atomicAdd(&hist[i], (unsigned long long)sh_hist[i]);
}

// ----------------------------------------------------------------------------- LSD radix sort
// The finite cells' keys, packed in any order: one global reservation per CTA and task, not per warp, since
// every CTA reserves from the same counter.
template <typename T, typename K>
__global__ void __launch_bounds__(kThreads) compact_keys_kernel(const char *__restrict__ in, int64_t in_pitch,
                                                                int64_t H, int64_t W, K *__restrict__ keys,
                                                                unsigned long long *__restrict__ count) {
    __shared__ unsigned warp_n[kWarps];
    __shared__ unsigned long long base;
    const CellKeys<T> src{in, in_pitch};
    const unsigned lane = threadIdx.x & 31, w = threadIdx.x >> 5, lt = (1u << lane) - 1u;
    for_each_chunk(H, W, [&](int64_t r, int64_t c0) {
        uint64_t key[kItems];
        unsigned take[kItems], before = 0, mine[kItems];
#pragma unroll
        for (int k = 0; k < kItems; ++k) {
            const int64_t c = c0 + k * kThreads;
            const bool ok = c < W && src.key(r, c, key[k]);
            take[k] = __ballot_sync(0xffffffffu, ok);
            mine[k] = before + __popc(take[k] & lt);
            before += __popc(take[k]);
        }
        if (lane == 0) warp_n[w] = before;
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned total = 0;
            for (int v = 0; v < kWarps; ++v) {
                const unsigned n = warp_n[v];
                warp_n[v] = total;
                total += n;
            }
            base = total ? atomicAdd(count, (unsigned long long)total) : 0ull;
        }
        __syncthreads();
        const unsigned long long at = base + warp_n[w];
#pragma unroll
        for (int k = 0; k < kItems; ++k)
            if ((take[k] >> lane) & 1u) keys[at + mine[k]] = (K)key[k];
        __syncthreads();
    });
}

// table[d * nblk + b] = the keys of block b's range whose digit at `lo` is d
template <typename K>
__global__ void __launch_bounds__(kThreads) sort_hist_kernel(const K *__restrict__ keys, int64_t n, int64_t per,
                                                             int lo, unsigned long long *__restrict__ table) {
    __shared__ unsigned h[256];
    h[threadIdx.x] = 0;
    __syncthreads();
    const int64_t b0 = (int64_t)blockIdx.x * per, b1 = min(n, b0 + per);
    const unsigned lane = threadIdx.x & 31;
    for (int64_t i0 = b0; i0 < b1; i0 += kThreads) {
        const int64_t i = i0 + threadIdx.x;
        count_warp(h, i < b1 ? (int)((keys[i] >> lo) & 255u) : -1, lane);
    }
    __syncthreads();
    table[(int64_t)threadIdx.x * gridDim.x + blockIdx.x] = h[threadIdx.x];
}

// exclusive scan of table[0 .. len) in one CTA
__global__ void __launch_bounds__(1024) sort_scan_kernel(unsigned long long *__restrict__ table, int64_t len) {
    __shared__ unsigned long long part[1024];
    const int64_t per = (len + 1023) / 1024, a = threadIdx.x * per, b = min(len, a + per);
    unsigned long long s = 0;
    for (int64_t i = a; i < b; ++i) s += table[i];
    part[threadIdx.x] = s;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
        const unsigned long long v = threadIdx.x >= (unsigned)o ? part[threadIdx.x - o] : 0ull;
        __syncthreads();
        part[threadIdx.x] += v;
        __syncthreads();
    }
    unsigned long long run = part[threadIdx.x] - s;
    for (int64_t i = a; i < b; ++i) {
        const unsigned long long v = table[i];
        table[i] = run;
        run += v;
    }
}

// The lanes whose d (0 .. 511) equals this lane's, from nine ballots
__device__ __forceinline__ unsigned match_digit(unsigned d) {
    unsigned peers = 0xffffffffu;
#pragma unroll
    for (int b = 0; b < 9; ++b) {
        const unsigned bit = (d >> b) & 1u, bal = __ballot_sync(0xffffffffu, bit);
        peers &= bit ? bal : ~bal;
    }
    return peers;
}

// Stable scatter of block b's range by the digit at `lo`.  Warp w takes tile positions [w 32 kSortItems,
// (w + 1) 32 kSortItems) in rounds of 32; a key's place among equal digits is the count before it in its warp
// (earlier rounds, then lower lanes), then the warps before it, then the tiles before it.
template <typename K>
__global__ void __launch_bounds__(kThreads) sort_scatter_kernel(const K *__restrict__ keys, K *__restrict__ out,
                                                                int64_t n, int64_t per, int lo,
                                                                const unsigned long long *__restrict__ table) {
    __shared__ unsigned cnt[kWarps][257];
    __shared__ unsigned long long base[256];
    base[threadIdx.x] = table[(int64_t)threadIdx.x * gridDim.x + blockIdx.x];
    const int64_t b0 = (int64_t)blockIdx.x * per, b1 = min(n, b0 + per);
    const unsigned lane = threadIdx.x & 31, w = threadIdx.x >> 5, lt = (1u << lane) - 1u;
    for (int64_t t0 = b0; t0 < b1; t0 += kSortTile) {
        for (int i = threadIdx.x; i < kWarps * 257; i += kThreads) (&cnt[0][0])[i] = 0;
        __syncthreads();
        K k[kSortItems];
        int d[kSortItems];
        unsigned loc[kSortItems];
#pragma unroll
        for (int j = 0; j < kSortItems; ++j) {
            const int64_t i = t0 + (int64_t)w * 32 * kSortItems + j * 32 + lane;
            k[j] = i < b1 ? keys[i] : K(0);
            d[j] = i < b1 ? (int)((k[j] >> lo) & 255u) : 256;
            const unsigned peers = match_digit(d[j]);
            loc[j] = cnt[w][d[j]] + __popc(peers & lt);
            __syncwarp();
            if (lane == (unsigned)(__ffs(peers) - 1)) cnt[w][d[j]] += __popc(peers);
            __syncwarp();
        }
        __syncthreads();
        {
            unsigned long long run = base[threadIdx.x];
            for (int v = 0; v < kWarps; ++v) {
                const unsigned c = cnt[v][threadIdx.x];
                cnt[v][threadIdx.x] = (unsigned)(run - base[threadIdx.x]);
                run += c;
            }
            __syncthreads();
#pragma unroll
            for (int j = 0; j < kSortItems; ++j)
                if (d[j] < 256) out[base[d[j]] + cnt[w][d[j]] + loc[j]] = k[j];
            __syncthreads();
            base[threadIdx.x] = run;
        }
    }
}

// ----------------------------------------------------------------------------- maximum_breaks picks
// mode 0: the unique keys of s, in any order.  mode 1: (s[i - 1], s[i]) for the gaps np.argsort(diffs,
// kind='stable')[-m:] selects: key above `tie`, or equal to it at a position >= pos.
template <typename T, typename K>
__global__ void __launch_bounds__(kThreads) pick_kernel(const K *__restrict__ s, int64_t n, int mode, uint64_t tie,
                                                        int64_t pos, K *__restrict__ out, int64_t cap,
                                                        unsigned long long *__restrict__ count) {
    const GapKeys<T, K> g{s};
    const unsigned lane = threadIdx.x & 31;
    for_each_chunk(1, n, [&](int64_t, int64_t c0) {
#pragma unroll
        for (int k = 0; k < kItems; ++k) {
            const int64_t i = c0 + k * kThreads;
            uint64_t gk = 0;
            bool ok = false;
            if (i < n) {
                if (mode == 0) ok = i == 0 || s[i] != s[i - 1];
                else ok = g.key(0, i, gk) && (gk > tie || (gk == tie && i >= pos));
            }
            const unsigned take = __ballot_sync(0xffffffffu, ok);
            unsigned long long b = 0;
            if (lane == 0 && take) b = atomicAdd(count, (unsigned long long)__popc(take));
            b = __shfl_sync(0xffffffffu, b, 0);
            const unsigned long long at = b + __popc(take & ((1u << lane) - 1u));
            if (ok && (int64_t)at < cap) {
                if (mode == 0) out[at] = s[i];
                else { out[2 * at] = s[i - 1]; out[2 * at + 1] = s[i]; }
            }
        }
    });
}

// ----------------------------------------------------------------------------- host helpers
int grid_for(int64_t H, int64_t W, int per_sm) {
    const int64_t tasks = H * ((W + kChunk - 1) / kChunk);
    return (int)std::max<int64_t>(1, std::min<int64_t>(tasks, (int64_t)sm_count() * per_sm));
}

// the sort's second key buffer, rounded up so that the digit table after it is aligned
int64_t keys_bytes(int64_t n, int64_t ksz) { return (n * ksz + 255) / 256 * 256; }

int key_bits(int dtype) {
    switch (dtype) {
        case XRS_F64: case XRS_I64: return 64;
        case XRS_I16: case XRS_U16: return 16;
        default: return 32;
    }
}

template <typename F> int with_cell_type(int dtype, F &&f) {
    switch (dtype) {
        case XRS_F32: return f(float{});
        case XRS_F64: return f(double{});
        case XRS_I32: return f(int32_t{});
        case XRS_I64: return f(int64_t{});
        case XRS_I16: return f(int16_t{});
        case XRS_U16: return f(uint16_t{});
        default: set_error("unknown cell type %d", dtype); return XRS_EINVAL;
    }
}

// The histogram of one digit pass over `src` for the sorted prefixes, copied to `host` (G x 256).
template <typename Src>
int select_pass(const Src &src, int64_t H, int64_t W, const std::vector<uint64_t> &prefixes, int lo,
                uint64_t *dprefix, unsigned long long *dhist, std::vector<unsigned long long> &host, cudaStream_t s) {
    const int G = (int)prefixes.size();
    const size_t smem = (size_t)G * 256 * sizeof(unsigned);
    XRS_CUDA(cudaFuncSetAttribute(select_hist_kernel<Src>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    XRS_CUDA(cudaMemcpyAsync(dprefix, prefixes.data(), G * sizeof(uint64_t), cudaMemcpyHostToDevice, s));
    XRS_CUDA(cudaMemsetAsync(dhist, 0, (size_t)G * 256 * sizeof(unsigned long long), s));
    const int per_sm = G <= 8 ? 8 : (G <= 32 ? 4 : 1);
    select_hist_kernel<Src><<<grid_for(H, W, per_sm), kThreads, smem, s>>>(src, H, W, dprefix, G, lo, dhist);
    XRS_CUDA(cudaGetLastError());
    host.resize((size_t)G * 256);
    XRS_CUDA(cudaMemcpyAsync(host.data(), dhist, host.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    XRS_CUDA(cudaStreamSynchronize(s));
    return XRS_OK;
}

// Radix select over `src`: first pass (the top digit) either run here or given in hist0; keys[i] / rem[i] = the
// ranks[i]-th smallest key and that rank less the keys below it.
template <typename Src>
int radix_select(const Src &src, int64_t H, int64_t W, int bits, const int64_t *ranks, int nr, uint64_t *keys,
                 int64_t *rem, int64_t *n_keys, uint64_t *hist0, void *scratch, cudaStream_t s) {
    uint64_t *dprefix = static_cast<uint64_t *>(scratch);
    unsigned long long *dhist = reinterpret_cast<unsigned long long *>(dprefix + kMaxGroups);
    std::vector<unsigned long long> h;
    int lo = bits - 8;
    if (nr == 0) {
        int rc = select_pass(src, H, W, std::vector<uint64_t>{0}, lo, dprefix, dhist, h, s);
        if (rc != XRS_OK) return rc;
        int64_t n = 0;
        for (int d = 0; d < 256; ++d) {
            hist0[d] = h[d];
            n += (int64_t)h[d];
        }
        *n_keys = n;
        return XRS_OK;
    }
    std::vector<uint64_t> pre(nr, 0);
    std::vector<int64_t> r(ranks, ranks + nr);
    h.assign(hist0, hist0 + 256);
    std::vector<uint64_t> groups{0};
    for (;;) {
        for (int i = 0; i < nr; ++i) {   // choose each target's digit in its group's histogram
            const int g = (int)(std::lower_bound(groups.begin(), groups.end(), pre[i]) - groups.begin());
            const unsigned long long *hg = h.data() + (size_t)g * 256;
            int d = 0;
            while (d < 255 && (unsigned long long)r[i] >= hg[d]) r[i] -= (int64_t)hg[d++];
            pre[i] = (pre[i] << 8) | (uint64_t)d;
        }
        if (lo == 0) break;
        lo -= 8;
        std::vector<uint64_t> all(pre);
        std::sort(all.begin(), all.end());
        all.erase(std::unique(all.begin(), all.end()), all.end());
        // more distinct prefixes than one launch holds: a pass per batch, each batch's targets updated alone
        std::vector<unsigned long long> merged(all.size() * 256);
        for (size_t b = 0; b < all.size(); b += kMaxGroups) {
            std::vector<uint64_t> part(all.begin() + b, all.begin() + std::min(all.size(), b + kMaxGroups));
            int rc = select_pass(src, H, W, part, lo, dprefix, dhist, h, s);
            if (rc != XRS_OK) return rc;
            std::copy(h.begin(), h.end(), merged.begin() + b * 256);
        }
        h.swap(merged);
        groups.swap(all);
    }
    for (int i = 0; i < nr; ++i) {
        keys[i] = pre[i];
        rem[i] = r[i];
    }
    return XRS_OK;
}

template <typename F> int with_key_type(int dtype, F &&f) {
    if (key_bits(dtype) == 64) return f(uint64_t{});
    return f(uint32_t{});
}

}  // namespace
}  // namespace xrs

using namespace xrs;

extern "C" {

int xrs_classify_cells(const void *in, int dtype, int64_t in_pitch, int64_t H, int64_t W, int member,
                       const double *bins, const float *new_values, int nb, void *out, int64_t out_pitch,
                       xrs_stream_t s) {
    XRS_REQUIRE(H >= 0 && W >= 0 && nb >= 0, "bad shape");
    if (H == 0 || W == 0) return XRS_OK;
    XRS_REQUIRE(in && out && (nb == 0 || (bins && (member || new_values))), "NULL pointer");
    const size_t esz = dtype == XRS_F64 || dtype == XRS_I64 ? 8 : (dtype == XRS_I16 || dtype == XRS_U16 ? 2 : 4);
    XRS_REQUIRE(in_pitch >= W * (int64_t)esz && out_pitch >= W * (int64_t)(member ? esz : 4), "pitch below the row");
    const size_t smem = (size_t)nb * (sizeof(double) + sizeof(float));
    const int in_smem = smem <= 96 * 1024 ? 1 : 0;   // else the lookup reads the table through L1 / L2
    const int64_t osz = member ? (int64_t)esz : 4;
    if (in_pitch == W * (int64_t)esz && out_pitch == W * osz) {   // contiguous: one row of H W cells
        W *= H;
        H = 1;
        in_pitch = W * (int64_t)esz;
        out_pitch = W * osz;
    }
    const int64_t span = 2 * kThreads * (16 / (int64_t)esz);
    const int64_t tasks = H * ((W + span - 1) / span);
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(tasks, (int64_t)sm_count() * 8));
    return with_cell_type(dtype, [&](auto t) -> int {
        using T = decltype(t);
        auto kern = member ? classify_cells_kernel<T, true> : classify_cells_kernel<T, false>;
        const size_t sm = in_smem ? smem : 0;
        if (sm > 48 * 1024) XRS_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
        return launch(kern, grid, kThreads, sm, (cudaStream_t)s, kClassify, (const char *)in, in_pitch, H, W, bins,
                      new_values, nb, in_smem, (char *)out, out_pitch);
    });
}

int xrs_classify_moments_scratch_bytes(int64_t *bytes) {
    XRS_REQUIRE(bytes, "NULL pointer");
    *bytes = (int64_t)sm_count() * 8 * (int64_t)sizeof(Moments);
    return XRS_OK;
}

int xrs_classify_moments(const void *in, int dtype, int64_t in_pitch, int64_t H, int64_t W, double above,
                         double *out5, void *scratch, int64_t scratch_bytes, xrs_stream_t s) {
    XRS_REQUIRE(H >= 0 && W >= 0, "bad shape");
    XRS_REQUIRE(out5 && scratch && (in || H * W == 0), "NULL pointer");
    XRS_REQUIRE(scratch_bytes >= (int64_t)sm_count() * 8 * (int64_t)sizeof(Moments), "scratch too small");
    const int grid = grid_for(H, W, 8);
    Moments *part = static_cast<Moments *>(scratch);
    int rc = with_cell_type(dtype, [&](auto t) -> int {
        using T = decltype(t);
        moments_kernel<T><<<grid, kThreads, 0, (cudaStream_t)s>>>((const char *)in, in_pitch, H, W, above, part);
        XRS_CUDA(cudaGetLastError());
        return XRS_OK;
    });
    if (rc != XRS_OK) return rc;
    moments_finish_kernel<<<1, kThreads, 0, (cudaStream_t)s>>>(part, grid, out5);
    XRS_CUDA(cudaGetLastError());
    return XRS_OK;
}

int xrs_classify_select_scratch_bytes(int64_t *bytes) {
    XRS_REQUIRE(bytes, "NULL pointer");
    *bytes = kMaxGroups * (int64_t)sizeof(uint64_t) + kMaxGroups * 256 * (int64_t)sizeof(unsigned long long);
    return XRS_OK;
}

int xrs_classify_select(int source, const void *in, int dtype, int64_t in_pitch, int64_t H, int64_t W, int bits,
                        uint64_t tie, const int64_t *ranks, int nr, uint64_t *keys, int64_t *rem, int64_t *n_keys,
                        uint64_t *hist0, void *scratch, int64_t scratch_bytes, xrs_stream_t s) {
    XRS_REQUIRE(H >= 0 && W >= 0 && nr >= 0, "bad shape");
    XRS_REQUIRE(bits >= 8 && bits <= 64 && bits % 8 == 0, "key bits must be 8 .. 64 in steps of 8");
    XRS_REQUIRE(source >= 0 && source <= 2, "unknown key source");
    XRS_REQUIRE(source == 0 || H == 1, "sorted keys are one row");
    XRS_REQUIRE(hist0 && scratch && (in || H * W == 0) && (nr == 0 || (ranks && keys && rem)) && (nr || n_keys),
                "NULL pointer");
    int64_t need = 0;
    xrs_classify_select_scratch_bytes(&need);
    XRS_REQUIRE(scratch_bytes >= need, "scratch too small");
    if (nr) {
        int64_t n = 0;
        for (int d = 0; d < 256; ++d) n += (int64_t)hist0[d];
        for (int i = 0; i < nr; ++i) XRS_REQUIRE(ranks[i] >= 0 && ranks[i] < n, "rank outside the keys");
    }
    cudaStream_t st = (cudaStream_t)s;
    return with_cell_type(dtype, [&](auto t) -> int {
        using T = decltype(t);
        if (source == 0)
            return radix_select(CellKeys<T>{(const char *)in, in_pitch}, H, W, bits, ranks, nr, keys, rem, n_keys,
                                hist0, scratch, st);
        return with_key_type(dtype, [&](auto kt) -> int {
            using K = decltype(kt);
            const GapKeys<T, K> g{static_cast<const K *>(in)};
            if (source == 1) return radix_select(g, H, W, bits, ranks, nr, keys, rem, n_keys, hist0, scratch, st);
            return radix_select(TiePositions<T, K>{g, tie}, H, W, bits, ranks, nr, keys, rem, n_keys, hist0, scratch,
                                st);
        });
    });
}

int xrs_classify_sort_scratch_bytes(int64_t n, int dtype, int64_t *bytes) {
    XRS_REQUIRE(bytes && n >= 0, "bad argument");
    const int64_t ksz = key_bits(dtype) == 64 ? 8 : 4;
    const int64_t nblk = (int64_t)sm_count() * 8;
    *bytes = keys_bytes(n, ksz) + 256 * nblk * 8 + 8;
    return XRS_OK;
}

int xrs_classify_sort(const void *in, int dtype, int64_t in_pitch, int64_t H, int64_t W, void *keys, int64_t *n_keys,
                      void *scratch, int64_t scratch_bytes, xrs_stream_t s) {
    XRS_REQUIRE(H >= 0 && W >= 0, "bad shape");
    XRS_REQUIRE(keys && scratch && n_keys && (in || H * W == 0), "NULL pointer");
    int64_t need = 0;
    xrs_classify_sort_scratch_bytes(H * W, dtype, &need);
    XRS_REQUIRE(scratch_bytes >= need, "scratch too small");
    cudaStream_t st = (cudaStream_t)s;
    const int bits = key_bits(dtype);
    return with_cell_type(dtype, [&](auto t) -> int {
        using T = decltype(t);
        return with_key_type(dtype, [&](auto kt) -> int {
            using K = decltype(kt);
            const int64_t ksz = sizeof(K), nblk_max = (int64_t)sm_count() * 8;
            K *alt = static_cast<K *>(scratch);
            unsigned long long *table = reinterpret_cast<unsigned long long *>((char *)scratch + keys_bytes(H * W, ksz));
            unsigned long long *count = table + 256 * nblk_max;
            XRS_CUDA(cudaMemsetAsync(count, 0, sizeof(unsigned long long), st));
            compact_keys_kernel<T, K><<<grid_for(H, W, 8), kThreads, 0, st>>>((const char *)in, in_pitch, H, W,
                                                                            (K *)keys, count);
            XRS_CUDA(cudaGetLastError());
            unsigned long long n = 0;
            XRS_CUDA(cudaMemcpyAsync(&n, count, sizeof(n), cudaMemcpyDeviceToHost, st));
            XRS_CUDA(cudaStreamSynchronize(st));
            *n_keys = (int64_t)n;
            if (n < 2) return XRS_OK;
            const int64_t nblk = std::min<int64_t>(nblk_max, ((int64_t)n + kSortTile - 1) / kSortTile);
            const int64_t per = (((int64_t)n + nblk - 1) / nblk + kSortTile - 1) / kSortTile * kSortTile;
            K *a = (K *)keys, *b = alt;
            for (int lo = 0; lo < bits; lo += 8) {   // an even number of passes: the result ends in `keys`
                sort_hist_kernel<K><<<(unsigned)nblk, kThreads, 0, st>>>(a, (int64_t)n, per, lo, table);
                XRS_CUDA(cudaGetLastError());
                sort_scan_kernel<<<1, 1024, 0, st>>>(table, 256 * nblk);
                XRS_CUDA(cudaGetLastError());
                sort_scatter_kernel<K><<<(unsigned)nblk, kThreads, 0, st>>>(a, b, (int64_t)n, per, lo, table);
                XRS_CUDA(cudaGetLastError());
                std::swap(a, b);
            }
            return XRS_OK;
        });
    });
}

int xrs_classify_pick(const void *sorted, int dtype, int64_t n, int mode, uint64_t tie, int64_t pos, void *out,
                      int64_t cap, int64_t *count, void *scratch, xrs_stream_t s) {
    XRS_REQUIRE(n >= 0 && cap >= 0 && (mode == 0 || mode == 1), "bad argument");
    XRS_REQUIRE(count && scratch && (sorted || n == 0) && (out || cap == 0), "NULL pointer");
    cudaStream_t st = (cudaStream_t)s;
    unsigned long long *dcount = static_cast<unsigned long long *>(scratch);
    XRS_CUDA(cudaMemsetAsync(dcount, 0, sizeof(unsigned long long), st));
    if (n) {
        int rc = with_cell_type(dtype, [&](auto t) -> int {
            using T = decltype(t);
            return with_key_type(dtype, [&](auto kt) -> int {
                using K = decltype(kt);
                pick_kernel<T, K><<<grid_for(1, n, 8), kThreads, 0, st>>>((const K *)sorted, n, mode, tie, pos,
                                                                        (K *)out, cap, dcount);
                XRS_CUDA(cudaGetLastError());
                return XRS_OK;
            });
        });
        if (rc != XRS_OK) return rc;
    }
    unsigned long long c = 0;
    XRS_CUDA(cudaMemcpyAsync(&c, dcount, sizeof(c), cudaMemcpyDeviceToHost, st));
    XRS_CUDA(cudaStreamSynchronize(st));
    *count = (int64_t)c;
    return XRS_OK;
}

}  // extern "C"

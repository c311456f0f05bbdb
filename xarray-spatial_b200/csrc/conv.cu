// conv.cu -- general k x k neighbourhood operators: convolve_2d (convolution.py:285-313) and
// the masked focal statistics behind focal.apply / focal_stats (focal.py:305-326, 268-302).
//
// One CTA (256 threads = 32 x 8) per 128 x 32 output tile, persistent over tiles.  The
// (tile + halo) block is brought into shared memory by TMA 2-D bulk loads with NaN
// out-of-bounds fill: for convolve_2d that produces the reference's NaN ring for free
// (NaN * w = NaN, even for w = 0), for the focal statistics out-of-raster cells are skipped
// exactly like NaN cells, which is the reference's clamped window.
//
// convolve_2d: the tile is widened to float64 once in shared memory; every thread owns a
// 4 x 4 block of outputs and accumulates in float64 with FMA (the reference accumulates
// `kernel(f64) * data(f32)` in a float64 `num`); weights are read from the kernel-parameter
// constant bank.  Bound: FP64 FMA rate for k >= 5 (2*k*k flop/cell), HBM for k = 3.
#include <stdlib.h>
#include <string.h>

#include <type_traits>
#include <vector>

#include "common.cuh"

namespace xrs {

constexpr int kMaxTaps = 2401;  // up to 49 x 49
constexpr int kTileW = 128, kTileH = 32;

struct ConvWeights {
    double w[kMaxTaps];
};
struct MaskBits {
    unsigned char m[kMaxTaps];
};

struct TileGeom {
    int64_t H, W;
    int kh, kw, ry, rx;
    int pad;       // cells loaded left of the tile: rx rounded up to 4 (TMA box starts must stay
                   // 16-byte aligned in the innermost dimension)
    int off;       // pad - rx: column offset of tap 0 inside the shared tile
    int sw;        // shared tile width (cells), multiple of 4
    int sh;        // shared tile height = kTileH + kh - 1
    int tiles_x, tiles_y;
    int box_h;     // rows per TMA box (sh is loaded in ceil(sh / box_h) boxes)
    __host__ __device__ size_t tile_cells() const { return (size_t)((sh + box_h - 1) / box_h) * box_h * sw; }
    size_t smem_bytes() const { return tile_cells() * sizeof(float) + 16; }   // the tile, then its mbarrier
};

// The persistent loop of the tiled kernels over kTileW x tile_h output tiles: CTA b takes tiles b, b + gridDim.x,
// ..., brings each (tile + halo) block into shared memory and runs body(tile32, x0, y0) on it.  Shared memory
// holds the block, then one mbarrier; thread 0 initialises the barrier and issues the TMA boxes, everyone waits
// on it.
template <typename F>
__device__ __forceinline__ void tile_loop(const CUtensorMap *tmap, const TileGeom &g, int tile_h, F &&body) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    float *tile32 = reinterpret_cast<float *>(smem_raw);
    uint64_t *bar = reinterpret_cast<uint64_t *>(smem_raw + g.tile_cells() * sizeof(float));
    if (threadIdx.x == 0) {
        tma_prefetch_desc(tmap);
        mbar_init(bar, 1);
        mbar_fence_init();
    }
    __syncthreads();
    const int64_t n_tiles = (int64_t)g.tiles_x * g.tiles_y;
    uint32_t parity = 0;
    for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const int tile_y = (int)(t / g.tiles_x), tile_x = (int)(t % g.tiles_x);
        const int x0 = tile_x * kTileW, y0 = tile_y * tile_h;
        if (threadIdx.x == 0) {
            const int nbox = (g.sh + g.box_h - 1) / g.box_h;
            mbar_arrive_expect_tx(bar, (uint32_t)(nbox * g.box_h * g.sw * sizeof(float)));
            for (int b = 0; b < nbox; ++b)
                tma_load_2d(tile32 + (size_t)b * g.box_h * g.sw, tmap, bar, x0 - g.pad, y0 - g.ry + b * g.box_h);
        }
        mbar_wait(bar, parity);
        parity ^= 1u;
        body(tile32, x0, y0);
        __syncthreads();  // the tile buffer is reused by the next iteration
    }
}

// ----------------------------------------------------------------------------- convolve
// 128 x 64 output tile per CTA, 256 threads = 16 (x) x 16 (y); a thread owns 4 rows x (4 + 4)
// columns: columns 4tx .. 4tx+3 and 64+4tx .. 64+4tx+3, so that consecutive lanes read
// consecutive 16-byte pieces of a shared-memory row (conflict-free LDS.128).  The float32 tile
// is read directly and widened in registers (16 F2F per 128 DFMA); 32 independent float64
// accumulators per thread give the FP64 pipe enough parallelism at 2-3 CTAs per SM.
constexpr int kConvTileH = 64;

// A thread's 4 x 8 outputs: rows y .. y + 3, columns xa .. xa + 3 and xa + 64 .. xa + 67.
__device__ __forceinline__ void store_tile32(float *out, int64_t pitch_elems, const TileGeom &g, int64_t y,
                                             int64_t xa, const double (&acc)[4][8]) {
    const int64_t xb = xa + 64;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const int64_t yo = y + r;
        if (yo < g.H) {  // W % 4 == 0 on this path: a float4 is all-in or all-out
            float *orow = out + yo * pitch_elems;
            if (xa < g.W)
                __stcs(reinterpret_cast<float4 *>(orow + xa),
                       make_float4((float)acc[r][0], (float)acc[r][1], (float)acc[r][2], (float)acc[r][3]));
            if (xb < g.W)
                __stcs(reinterpret_cast<float4 *>(orow + xb),
                       make_float4((float)acc[r][4], (float)acc[r][5], (float)acc[r][6], (float)acc[r][7]));
        }
    }
}

// KW > 0: kernel width known at compile time (5, 7, 9: the usual custom kernels) -- the tap-chunk
// loop unrolls and its chunk / tap tests fold away; KW == 0: any odd shape.
template <int KW>
__global__ void __launch_bounds__(256)
conv2d_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ ConvWeights cw,
              float *__restrict__ out, int64_t out_pitch_elems, const TileGeom g) {
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    tile_loop(&tmap, g, kConvTileH, [&](const float *tile32, int x0, int y0) {
        double acc[4][8];
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int c = 0; c < 8; ++c) acc[r][c] = 0.0;

        // Input row j of the thread's window feeds output row r with kernel row ky = j - r.
        // Rows 3 .. kh-1 feed all four output rows, and 4-tap chunks lying fully inside the
        // kernel need no tap test: that common case is straight-line DFMA code; the few edge
        // rows / edge chunks take the generic, predicated path.  Taps are indexed from the
        // 16-byte aligned tile origin: tap kx sits at column kx + off.
        const int rows_in = 4 + g.kh - 1;
        constexpr int kOffC = KW ? ((KW / 2 + 3) / 4 * 4 - KW / 2) : 0;
        const int kw = KW ? KW : g.kw;
        const int off = KW ? kOffC : g.off;
        const int n_taps = off + kw;
        for (int j = 0; j < rows_in; ++j) {
            const float *rowp = tile32 + (size_t)(ty * 4 + j) * g.sw + 4 * tx;
            const bool full_rows = (j >= 3) && (j < g.kh);
            auto chunk = [&](const int kb) {
                const float4 a0 = *reinterpret_cast<const float4 *>(rowp + kb);
                const float4 a1 = *reinterpret_cast<const float4 *>(rowp + kb + 4);
                const float4 b0 = *reinterpret_cast<const float4 *>(rowp + 64 + kb);
                const float4 b1 = *reinterpret_cast<const float4 *>(rowp + 64 + kb + 4);
                const double va[8] = {(double)a0.x, (double)a0.y, (double)a0.z, (double)a0.w,
                                      (double)a1.x, (double)a1.y, (double)a1.z, (double)a1.w};
                const double vb[8] = {(double)b0.x, (double)b0.y, (double)b0.z, (double)b0.w,
                                      (double)b1.x, (double)b1.y, (double)b1.z, (double)b1.w};
                const bool full_chunk = (kb >= off) && (kb + 4 <= n_taps);
                if (full_chunk && full_rows) {
                    const double *w0 = cw.w + (j * kw + kb - off);  // kernel row j, taps kb-off ..
#pragma unroll
                    for (int r = 0; r < 4; ++r) {
                        const double *wr = w0 - r * kw;            // kernel row j - r
#pragma unroll
                        for (int tt = 0; tt < 4; ++tt) {
                            const double wv = wr[tt];
#pragma unroll
                            for (int c = 0; c < 4; ++c) {
                                acc[r][c] = fma(wv, va[c + tt], acc[r][c]);
                                acc[r][4 + c] = fma(wv, vb[c + tt], acc[r][4 + c]);
                            }
                        }
                    }
                } else if (full_chunk) {
                    // lead-in / lead-out rows of the window: some output rows have no kernel row here
                    const double *w0 = cw.w + (j * kw + kb - off);
#pragma unroll
                    for (int r = 0; r < 4; ++r) {
                        if (j - r >= 0 && j - r < g.kh) {  // warp-uniform
                            const double *wr = w0 - r * kw;        // kernel row j - r
#pragma unroll
                            for (int tt = 0; tt < 4; ++tt) {
                                const double wv = wr[tt];
#pragma unroll
                                for (int c = 0; c < 4; ++c) {
                                    acc[r][c] = fma(wv, va[c + tt], acc[r][c]);
                                    acc[r][4 + c] = fma(wv, vb[c + tt], acc[r][4 + c]);
                                }
                            }
                        }
                    }
                } else {
#pragma unroll
                    for (int r = 0; r < 4; ++r) {
                        const int ky = j - r;
                        if (ky >= 0 && ky < g.kh) {
#pragma unroll
                            for (int tt = 0; tt < 4; ++tt) {
                                const int kx = kb + tt - off;
                                if (kx >= 0 && kx < kw) {
                                    const double wv = cw.w[ky * kw + kx];
#pragma unroll
                                    for (int c = 0; c < 4; ++c) {
                                        acc[r][c] = fma(wv, va[c + tt], acc[r][c]);
                                        acc[r][4 + c] = fma(wv, vb[c + tt], acc[r][4 + c]);
                                    }
                                }
                            }
                        }
                    }
                }
            };
            if constexpr (KW > 0) {
#pragma unroll
                for (int kb = 0; kb < kOffC + KW; kb += 4) chunk(kb);
            } else {
                for (int kb = 0; kb < n_taps; kb += 4) chunk(kb);
            }
        }
        store_tile32(out, out_pitch_elems, g, (int64_t)y0 + ty * 4, (int64_t)x0 + 4 * tx, acc);
    });
}

// Square K x K kernels with K in {5, 7, ..., 13} (the usual hand-made filters; at K = 15 the
// unrolled code no longer fits the instruction cache and the looped kernel is faster): everything is unrolled,
// so each loaded cell is widened to float64 once per row (not once per tap chunk) and every
// weight is an immediate constant-bank operand of its DFMA.  Same tile / thread layout and
// the same per-output accumulation order (row-major taps) as conv2d_kernel.
template <int K>
__global__ void __launch_bounds__(256, 2)
conv2d_fixed_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ ConvWeights cw,
                    float *__restrict__ out, int64_t out_pitch_elems, const TileGeom g) {
    constexpr int kOff = (K / 2 + 3) / 4 * 4 - K / 2;   // column of tap 0 relative to the aligned origin
    constexpr int kVals = (kOff + K + 3 + 3) / 4 * 4;   // cells a thread needs per row and half
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    tile_loop(&tmap, g, kConvTileH, [&](const float *tile32, int x0, int y0) {
        double acc[4][8];
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int c = 0; c < 8; ++c) acc[r][c] = 0.0;
        const float *base = tile32 + (size_t)(ty * 4) * g.sw + 4 * tx;
#pragma unroll
        for (int j = 0; j < K + 3; ++j) {
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                const float *rowp = base + (size_t)j * g.sw + half * 64;
                double d[kVals];
#pragma unroll
                for (int q = 0; q < kVals / 4; ++q) {
                    const float4 f = *reinterpret_cast<const float4 *>(rowp + 4 * q);
                    d[4 * q + 0] = (double)f.x; d[4 * q + 1] = (double)f.y;
                    d[4 * q + 2] = (double)f.z; d[4 * q + 3] = (double)f.w;
                }
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    const int ky = j - r;
                    if (ky >= 0 && ky < K) {
#pragma unroll
                        for (int kx = 0; kx < K; ++kx) {
                            const double wv = cw.w[ky * K + kx];
#pragma unroll
                            for (int c = 0; c < 4; ++c)
                                acc[r][half * 4 + c] = fma(wv, d[c + kx + kOff], acc[r][half * 4 + c]);
                        }
                    }
                }
            }
        }
        store_tile32(out, out_pitch_elems, g, (int64_t)y0 + ty * 4, (int64_t)x0 + 4 * tx, acc);
    });
}

// Fallback for rasters TMA cannot describe: one thread per cell, bounds-checked loads.
__global__ void __launch_bounds__(256)
conv2d_direct_kernel(const float *__restrict__ in, int64_t in_pitch_elems, const __grid_constant__ ConvWeights cw,
                     float *__restrict__ out, int64_t out_pitch_elems, int64_t H, int64_t W, int kh, int kw) {
    const int64_t n = H * W;
    const int ry = kh / 2, rx = kw / 2;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t y = i / W, x = i % W;
        double acc = 0.0;
        for (int ky = 0; ky < kh; ++ky)
            for (int kx = 0; kx < kw; ++kx) {
                const int64_t yy = y + ky - ry, xx = x + kx - rx;
                const double v = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? (double)in[yy * in_pitch_elems + xx]
                                                                            : nan_of<double>();
                acc = fma(cw.w[ky * kw + kx], v, acc);
            }
        out[y * out_pitch_elems + x] = (float)acc;
    }
}

// ----------------------------------------------------------------------------- focal statistics
// Reducers follow Numba's nan-functions (numba/np/arraymath.py) as used by focal.py:268-302:
// mean/var/std accumulate in f64 (var two-pass about the f64 mean), sum accumulates in f32 in
// row-major window order (bit-identical to np.nansum on the f32 scratch), min/max skip NaN.
// Numba's nanmin / nanmax step: replace unless strictly ordered, so a NaN accumulator takes the first
// non-NaN cell, a NaN cell never replaces, and among equal cells (-0.0 and +0.0) the LAST in window order
// wins.  fminf / fmaxf would differ in the sign bit: they order -0.0 below +0.0.
__device__ __forceinline__ void nan_min_step(float &mn, float v) {
    if (v == v && !(mn < v)) mn = v;
}
__device__ __forceinline__ void nan_max_step(float &mx, float v) {
    if (v == v && !(mx > v)) mx = v;
}
template <typename Fetch>
__device__ __forceinline__ float focal_reduce(const Fetch &fetch, const MaskBits &mask, int kh, int kw, int stat) {
    if (stat == XRS_STAT_MEAN || stat == XRS_STAT_VAR || stat == XRS_STAT_STD) {
        double c = 0.0;
        int cnt = 0;
        for (int ky = 0; ky < kh; ++ky)
            for (int kx = 0; kx < kw; ++kx)
                if (mask.m[ky * kw + kx]) {
                    const float v = fetch(ky, kx);
                    if (v == v) { c += (double)v; ++cnt; }
                }
        const double m = c / (double)cnt;
        if (stat == XRS_STAT_MEAN) return (float)m;
        double ssd = 0.0;
        for (int ky = 0; ky < kh; ++ky)
            for (int kx = 0; kx < kw; ++kx)
                if (mask.m[ky * kw + kx]) {
                    const float v = fetch(ky, kx);
                    if (v == v) { const double d = (double)v - m; ssd += d * d; }
                }
        const double var = ssd / (double)cnt;
        return (float)(stat == XRS_STAT_VAR ? var : sqrt(var));
    } else if (stat == XRS_STAT_SUM) {
        float c = 0.f;
        for (int ky = 0; ky < kh; ++ky)
            for (int kx = 0; kx < kw; ++kx)
                if (mask.m[ky * kw + kx]) {
                    const float v = fetch(ky, kx);
                    if (v == v) c += v;
                }
        return c;
    } else {
        // nanmin / nanmax start from scratch[0] (NaN unless the first window cell takes part)
        float mn = nan_of<float>(), mx = nan_of<float>();
        for (int ky = 0; ky < kh; ++ky)
            for (int kx = 0; kx < kw; ++kx)
                if (mask.m[ky * kw + kx]) {
                    const float v = fetch(ky, kx);
                    nan_min_step(mn, v);
                    nan_max_step(mx, v);
                }
        return stat == XRS_STAT_MIN ? mn : stat == XRS_STAT_MAX ? mx : mx - mn;
    }
}

// One loaded window cell as the reducers see it: NaN test, f64 widening and the "skip NaN" masking
// happen once per loaded cell, not once per (output, tap) use.
struct FocalCell {
    float v;      // raw value
    float vz;     // value, 0 when NaN
    double d;     // (double)value
    double dz;    // (double)value, 0 when NaN
    int one;      // 1 when not NaN
    bool ok;
};

// The 8 cells of a 4-tap chunk: two 16-byte loads from p.
__device__ __forceinline__ void load_cells(const float *p, FocalCell (&cell)[8]) {
    const float4 q0 = *reinterpret_cast<const float4 *>(p);
    const float4 q1 = *reinterpret_cast<const float4 *>(p + 4);
    const float v[8] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        cell[i].v = v[i];
        cell[i].ok = (v[i] == v[i]);
        cell[i].vz = cell[i].ok ? v[i] : 0.f;
        cell[i].d = (double)v[i];
        cell[i].dz = (double)cell[i].vz;
        cell[i].one = cell[i].ok ? 1 : 0;
    }
}

// The output planes of the focal statistics.
struct StatPlanes {
    float *p[7];  // indexed by xrs_focal_stat; nullptr = not requested
};
constexpr int kAllStats = -1;  // as a kernel's statistic: every statistic whose plane is set

// The tiled kernel's output: the plane of its one statistic, or every plane for kAllStats.
template <int STAT>
using FocalOut = std::conditional_t<STAT == kAllStats, StatPlanes, float *__restrict__>;
template <int STAT>
FocalOut<STAT> focal_out(const StatPlanes &planes) {
    if constexpr (STAT == kAllStats) return planes;
    else return planes.p[STAT];
}
__device__ __forceinline__ float *plane_of(const StatPlanes &out, int s) { return out.p[s]; }
__device__ __forceinline__ float *plane_of(float *out, int) { return out; }

// The statistics of a thread's 4 x 4 outputs, for the tiled and the wide kernels alike.  STAT is one
// xrs_focal_stat, or kAllStats for every statistic whose plane in `out` is set.  sweep(f) calls f(r, c, cell) for
// every window cell of output (r, c), in row-major window order; store(plane, res) writes 4 x 4 results.
// Sweep A accumulates the float64 sum and the count (mean, var, std) and the float32 row-major sum (sum); sweep B
// the squared deviations about the float64 mean (var, std).  min and max (min, max, range) go into sweep A when
// kMinMaxInA, into sweep B otherwise: which is cheaper depends on the memory path.  A sweep with nothing to
// accumulate does not run: for one statistic that is known at compile time, for kAllStats the planes decide.
template <int STAT, bool kMinMaxInA, typename Out, typename Sweep, typename Store>
__device__ __forceinline__ void focal_outputs(const Out &out, const Sweep &sweep, const Store &store) {
    constexpr bool kAll = STAT == kAllStats;
    constexpr bool kMean = kAll || STAT == XRS_STAT_MEAN || STAT == XRS_STAT_VAR || STAT == XRS_STAT_STD;
    constexpr bool kSum = kAll || STAT == XRS_STAT_SUM;
    constexpr bool kMinMax = kAll || STAT == XRS_STAT_MIN || STAT == XRS_STAT_MAX || STAT == XRS_STAT_RANGE;
    constexpr bool kSsd = kAll || STAT == XRS_STAT_VAR || STAT == XRS_STAT_STD;
    auto want = [&](int s) { return kAll ? plane_of(out, s) != nullptr : STAT == s; };
    float res[4][4];
    double mean[4][4];
    int cnt[4][4];
    float fsum[4][4], mn[4][4], mx[4][4];
    double ssd[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c)
            mean[r][c] = 0.0, cnt[r][c] = 0, fsum[r][c] = 0.f, mn[r][c] = mx[r][c] = nan_of<float>();
    auto min_max = [&](int r, int c, const FocalCell &q) {
        nan_min_step(mn[r][c], q.v);
        nan_max_step(mx[r][c], q.v);
    };
    auto store_min_max = [&] {
        if (want(XRS_STAT_MIN)) store(plane_of(out, XRS_STAT_MIN), mn);
        if (want(XRS_STAT_MAX)) store(plane_of(out, XRS_STAT_MAX), mx);
        if (want(XRS_STAT_RANGE)) {
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c) res[r][c] = mx[r][c] - mn[r][c];
            store(plane_of(out, XRS_STAT_RANGE), res);
        }
    };
    if constexpr (kMean || kSum || (kMinMaxInA && kMinMax))
        sweep([&](int r, int c, const FocalCell &q) {  // sweep A
            if (kMean) mean[r][c] += q.dz, cnt[r][c] += q.one;
            if (kSum) fsum[r][c] += q.vz;
            if (kMinMaxInA && kMinMax) min_max(r, c, q);
        });
    if (want(XRS_STAT_SUM)) store(plane_of(out, XRS_STAT_SUM), fsum);
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            mean[r][c] = mean[r][c] / (double)cnt[r][c];
            res[r][c] = (float)mean[r][c];
        }
    if (want(XRS_STAT_MEAN)) store(plane_of(out, XRS_STAT_MEAN), res);
    if constexpr (kMinMaxInA) store_min_max();
    constexpr bool kMinMaxInB = !kMinMaxInA && kMinMax;
    if constexpr (kSsd || kMinMaxInB) {
        if ((kMinMaxInB && (want(XRS_STAT_MIN) || want(XRS_STAT_MAX) || want(XRS_STAT_RANGE))) || want(XRS_STAT_VAR) ||
            want(XRS_STAT_STD)) {
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c) ssd[r][c] = 0.0;
            sweep([&](int r, int c, const FocalCell &q) {  // sweep B
                if (kSsd) {
                    const double d = q.d - mean[r][c];
                    ssd[r][c] += q.ok ? d * d : 0.0;
                }
                if (kMinMaxInB) min_max(r, c, q);
            });
            if constexpr (kMinMaxInB) store_min_max();
            if (want(XRS_STAT_VAR) || want(XRS_STAT_STD)) {
#pragma unroll
                for (int r = 0; r < 4; ++r)
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        ssd[r][c] = ssd[r][c] / (double)cnt[r][c];
                        res[r][c] = (float)ssd[r][c];
                    }
                if (want(XRS_STAT_VAR)) store(plane_of(out, XRS_STAT_VAR), res);
                if (want(XRS_STAT_STD)) {
#pragma unroll
                    for (int r = 0; r < 4; ++r)
#pragma unroll
                        for (int c = 0; c < 4; ++c) res[r][c] = (float)sqrt(ssd[r][c]);
                    store(plane_of(out, XRS_STAT_STD), res);
                }
            }
        }
    }
}

// Register-blocked like conv2d_kernel: a thread owns 4 x 4 outputs, walks the input rows of its
// window once per sweep, loads 8 cells per 4-tap chunk with two LDS.128 and feeds every (output row,
// tap) pair whose mask bit is set.  Taps are visited in row-major window order for each output, so
// the float32 `sum` is bit-identical to np.nansum on the scratch.
template <typename F>
__device__ __forceinline__ void focal_sweep(const float *tile32, const MaskBits &mask, const TileGeom &g, int tx,
                                            int ty, F &&f) {
    const int rows_in = 4 + g.kh - 1;
    const int n_taps = g.off + g.kw;
    for (int j = 0; j < rows_in; ++j) {
        const float *rowp = tile32 + (size_t)(ty * 4 + j) * g.sw + 4 * tx;
        for (int kb = 0; kb < n_taps; kb += 4) {
            FocalCell cell[8];
            load_cells(rowp + kb, cell);
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int ky = j - r;
                if (ky >= 0 && ky < g.kh) {
#pragma unroll
                    for (int tt = 0; tt < 4; ++tt) {
                        const int kx = kb + tt - g.off;
                        if (kx >= 0 && kx < g.kw && mask.m[ky * g.kw + kx]) {  // warp-uniform
#pragma unroll
                            for (int c = 0; c < 4; ++c) f(r, c, cell[c + tt]);
                        }
                    }
                }
            }
        }
    }
}

__device__ __forceinline__ void store_tile16(float *plane, int64_t pitch_elems, int64_t H, int64_t W, int64_t y0,
                                             int64_t xo, const float (&res)[4][4]) {
#pragma unroll
    for (int r = 0; r < 4; ++r)
        if (y0 + r < H && xo < W)  // W % 4 == 0 on this path
            __stcs(reinterpret_cast<float4 *>(plane + (y0 + r) * pitch_elems + xo),
                   make_float4(res[r][0], res[r][1], res[r][2], res[r][3]));
}

// One statistic, or (kAllStats) every requested statistic in ONE pass over the raster: focal.focal_stats
// (focal.py:800-878) is seven `apply` calls stacked with xr.concat; here the tile is loaded once, the fused
// kernel runs 2 sweeps instead of 9, and each statistic goes straight into its plane of the (stats, y, x)
// result, with no stacking copy.  min and max are accumulated in sweep B.
template <int STAT>
__global__ void __launch_bounds__(256, STAT == kAllStats ? 2 : 0)
focal_tile_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ MaskBits mask,
                  const FocalOut<STAT> out, int64_t out_pitch_elems, const TileGeom g) {
    tile_loop(&tmap, g, kTileH, [&](const float *tile32, int x0, int y0) {
        const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
        auto sweep = [&](auto &&f) { focal_sweep(tile32, mask, g, tx, ty, f); };
        // Where the store coordinates are computed steers register allocation: before the sweeps the fused kernel
        // runs about 2 % faster, after them the single-statistic kernels need up to 6 fewer registers.
        if constexpr (STAT == kAllStats) {
            const int64_t xo = (int64_t)x0 + 4 * tx, yo = (int64_t)y0 + ty * 4;
            focal_outputs<STAT, false>(out, sweep, [&](float *plane, const float (&res)[4][4]) {
                store_tile16(plane, out_pitch_elems, g.H, g.W, yo, xo, res);
            });
        } else {
            focal_outputs<STAT, false>(out, sweep, [&](float *plane, const float (&res)[4][4]) {
                const int64_t xo = (int64_t)x0 + 4 * tx, yo = (int64_t)y0 + ty * 4;
                store_tile16(plane, out_pitch_elems, g.H, g.W, yo, xo, res);
            });
        }
    });
}

__global__ void __launch_bounds__(256)
focal_stat_direct_kernel(const float *__restrict__ in, int64_t in_pitch_elems, const __grid_constant__ MaskBits mask,
                         float *__restrict__ out, int64_t out_pitch_elems, int64_t H, int64_t W, int kh, int kw,
                         int stat) {
    const int64_t n = H * W;
    const int ry = kh / 2, rx = kw / 2;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t y = i / W, x = i % W;
        auto fetch = [=](int ky, int kx) {
            const int64_t yy = y + ky - ry, xx = x + kx - rx;
            return (yy >= 0 && yy < H && xx >= 0 && xx < W) ? in[yy * in_pitch_elems + xx] : nan_of<float>();
        };
        out[y * out_pitch_elems + x] = focal_reduce(fetch, mask, kh, kw, stat);
    }
}

// ----------------------------------------------------------------------------- wide windows
// Windows beyond the tiled kernels' reach (more than kMaxTaps taps, or a side above 63): the weights and
// the mask no longer fit the kernel-parameter bank, and the (tile + halo) block no longer fits shared
// memory.  A CTA owns 4 output rows x kWideConvW (convolve) or kWideStatW (statistics) columns and streams
// the kh + 3 input rows of its window through a ring of kRing shared-memory rows, filled by bounds-checked
// cp.async loads (any pitch, offset or width; out-of-raster cells NaN).  Input row J feeds output row r
// with kernel row J - r, uniform across the CTA, so every output receives its taps in row-major order,
// like the tiled kernels, and a thread's 4 x 8 (convolve) or 4 x 4 (statistics) outputs share each
// loaded cell.  The weights (kh rows of kwp doubles) and the mask (per kernel row: the [lo, hi) span of
// its ones and a bit row) live in a stream-ordered device buffer made for the call.
constexpr int kWideSide = 2047;
constexpr int kWideConvW = 2048, kWideStatW = 1024, kRing = 4;

struct WideGeom {
    int64_t H, W, in_pitch, out_pitch;  // pitches in cells
    int kh, kw;
    int kwp;                            // kw rounded up to 4: weight row stride, and the chunk loops' bound
    int nw;                             // mask words per kernel row
    int rw;                             // cells per ring row (multiple of 4)
    int tiles_x;
    int64_t n_tiles;
};

__device__ __forceinline__ void cp_async4(float *dst, const float *src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// Raster row y, columns xs .. xs + rw - 1, into ring row `slot`; out-of-raster cells are NaN.
__device__ __forceinline__ void ring_load(float *ring, const float *__restrict__ in, const WideGeom &g, int64_t y,
                                          int64_t xs, int slot) {
    float *dst = ring + (size_t)slot * g.rw;
    const bool row_in = y >= 0 && y < g.H;
    for (int i = threadIdx.x; i < g.rw; i += blockDim.x) {
        const int64_t x = xs + i;
        if (row_in && x >= 0 && x < g.W) cp_async4(dst + i, in + y * g.in_pitch + x);
        else dst[i] = nan_of<float>();
    }
}

// Streams input rows J = 0 .. kh + 2 (raster rows y0 - kh/2 + J) through the ring, kRing - 1 rows ahead of
// the one `fn(J, row)` consumes.
template <typename F>
__device__ __forceinline__ void ring_sweep(float *ring, const float *__restrict__ in, const WideGeom &g, int64_t y0,
                                           int64_t xs, F &&fn) {
    const int rows = g.kh + 3;
    const int64_t ya = y0 - g.kh / 2;
#pragma unroll
    for (int j = 0; j < kRing - 1; ++j) {
        if (j < rows) ring_load(ring, in, g, ya + j, xs, j);
        cp_async_commit();
    }
    for (int j = 0; j < rows; ++j) {
        cp_async_wait<kRing - 2>();
        __syncthreads();  // row j has landed everywhere, and every thread is done with row j - 1
        if (j + kRing - 1 < rows) ring_load(ring, in, g, ya + j + kRing - 1, xs, (j + kRing - 1) % kRing);
        cp_async_commit();
        fn(j, ring + (size_t)(j % kRing) * g.rw);
    }
    __syncthreads();  // the next sweep refills the ring
}

// A thread owns output rows y0 .. y0 + 3 and columns base + 0..3 and base + 64 + 0..3: consecutive lanes read
// consecutive 16-byte pieces of a ring row (conflict-free LDS.128), as in conv2d_kernel.
__global__ void __launch_bounds__(256)
conv2d_wide_kernel(const float *__restrict__ in, const double *__restrict__ w, float *__restrict__ out,
                   const WideGeom g) {
    extern __shared__ __align__(16) float ring[];
    const int base = 128 * (threadIdx.x >> 4) + 4 * (threadIdx.x & 15);
    const int kw4 = g.kw & ~3;
    for (int64_t t = blockIdx.x; t < g.n_tiles; t += gridDim.x) {
        const int64_t y0 = t / g.tiles_x * 4, x0 = t % g.tiles_x * kWideConvW;
        double acc[4][8];
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int c = 0; c < 8; ++c) acc[r][c] = 0.0;
        ring_sweep(ring, in, g, y0, x0 - g.kw / 2, [&](int j, const float *row) {
            const float *rowp = row + base;
            // taps kb .. kb + nt - 1 of the kernel rows j - r, one half of the thread's columns at a time.  Each
            // cell is widened once per chunk: left alone, the compiler sinks the F2F.F64 into every kernel-row
            // branch, and F2F.F64 issues at a quarter of the DFMA rate; the empty asm pins the widened value.
            auto chunk = [&](const int kb, const int nt) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const float4 a0 = *reinterpret_cast<const float4 *>(rowp + 64 * h + kb);
                    const float4 a1 = *reinterpret_cast<const float4 *>(rowp + 64 * h + kb + 4);
                    double v[8] = {(double)a0.x, (double)a0.y, (double)a0.z, (double)a0.w,
                                   (double)a1.x, (double)a1.y, (double)a1.z, (double)a1.w};
#pragma unroll
                    for (int i = 0; i < 8; ++i) asm("" : "+d"(v[i]));
#pragma unroll
                    for (int r = 0; r < 4; ++r) {
                        const int ky = j - r;
                        if (ky >= 0 && ky < g.kh) {  // CTA-uniform
                            const double2 *wr = reinterpret_cast<const double2 *>(w + (int64_t)ky * g.kwp + kb);
                            const double2 w01 = __ldg(wr), w23 = __ldg(wr + 1);
                            const double wv[4] = {w01.x, w01.y, w23.x, w23.y};
#pragma unroll
                            for (int tt = 0; tt < 4; ++tt)
                                if (tt < nt)
#pragma unroll
                                    for (int c = 0; c < 4; ++c)
                                        acc[r][4 * h + c] = fma(wv[tt], v[c + tt], acc[r][4 * h + c]);
                        }
                    }
                }
            };
            for (int kb = 0; kb < kw4; kb += 4) chunk(kb, 4);
            if (kw4 < g.kw) chunk(kw4, g.kw - kw4);
        });
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int64_t yo = y0 + r;
            if (yo >= g.H) continue;
            float *orow = out + yo * g.out_pitch;
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                const int64_t xo = x0 + base + (c & 3) + (c >> 2) * 64;
                if (xo < g.W) orow[xo] = (float)acc[r][c];
            }
        }
    }
}

// The statistics of focal_tile_kernel over a wide window (focal_outputs, with min and max in sweep A), a thread's
// 4 x 4 outputs being columns base .. base + 3.  Each sweep visits, per input row, only the 4-tap chunks inside
// the union of the spans of ones of the (up to four) kernel rows it feeds.
template <int STAT>
__global__ void __launch_bounds__(256)
focal_wide_kernel(const float *__restrict__ in, const int2 *__restrict__ span, const uint32_t *__restrict__ bits,
                  const StatPlanes planes, const WideGeom g) {
    extern __shared__ __align__(16) float ring[];
    const int base = 4 * threadIdx.x;
    for (int64_t t = blockIdx.x; t < g.n_tiles; t += gridDim.x) {
        const int64_t y0 = t / g.tiles_x * 4, x0 = t % g.tiles_x * kWideStatW, xs = x0 - g.kw / 2;
        auto sweep = [&](auto &&f) {
            ring_sweep(ring, in, g, y0, xs, [&](int j, const float *row) {
                const float *rowp = row + base;
                int lo = g.kwp, hi = 0;
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    const int ky = j - r;
                    if (ky >= 0 && ky < g.kh) {
                        const int2 sp = __ldg(span + ky);
                        lo = min(lo, sp.x);
                        hi = max(hi, sp.y);
                    }
                }
                for (int kb = lo; kb < hi; kb += 4) {
                    // load_cells written out: through the function, the compiler allocates this kernel's registers
                    // differently and the fused and var / std instantiations need 2 more
                    const float4 q0 = *reinterpret_cast<const float4 *>(rowp + kb);
                    const float4 q1 = *reinterpret_cast<const float4 *>(rowp + kb + 4);
                    const float v[8] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
                    FocalCell cell[8];
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        cell[i].v = v[i];
                        cell[i].ok = (v[i] == v[i]);
                        cell[i].vz = cell[i].ok ? v[i] : 0.f;
                        cell[i].d = (double)v[i];
                        cell[i].dz = (double)cell[i].vz;
                        cell[i].one = cell[i].ok ? 1 : 0;
                    }
#pragma unroll
                    for (int r = 0; r < 4; ++r) {
                        const int ky = j - r;
                        if (ky < 0 || ky >= g.kh) continue;
                        const uint32_t nib = (__ldg(bits + (int64_t)ky * g.nw + (kb >> 5)) >> (kb & 31)) & 15u;
                        if (nib == 15u) {  // CTA-uniform
#pragma unroll
                            for (int tt = 0; tt < 4; ++tt)
#pragma unroll
                                for (int c = 0; c < 4; ++c) f(r, c, cell[c + tt]);
                        } else if (nib) {
#pragma unroll
                            for (int tt = 0; tt < 4; ++tt)
                                if (nib >> tt & 1u)
#pragma unroll
                                    for (int c = 0; c < 4; ++c) f(r, c, cell[c + tt]);
                        }
                    }
                }
            });
        };
        focal_outputs<STAT, true>(planes, sweep, [&](float *plane, const float (&res)[4][4]) {
#pragma unroll
            for (int r = 0; r < 4; ++r)
                if (y0 + r < g.H)
#pragma unroll
                    for (int c = 0; c < 4; ++c)
                        if (x0 + base + c < g.W) plane[(y0 + r) * g.out_pitch + x0 + base + c] = res[r][c];
        });
    }
}

int check_window(int kh, int kw) {
    XRS_REQUIRE(kh >= 1 && kw >= 1 && (kh & 1) && (kw & 1), "kernel dimensions must be odd");
    XRS_REQUIRE(kh <= kWideSide && kw <= kWideSide, "kernel too large (max 2047 cells per side)");
    return XRS_OK;
}

static bool is_wide(int kh, int kw) { return kh * kw > kMaxTaps || kh > 63 || kw > 63; }

static WideGeom wide_geom(int64_t in_pitch, int64_t out_pitch, int64_t H, int64_t W, int kh, int kw, int tile_w) {
    WideGeom g;
    g.H = H; g.W = W; g.in_pitch = in_pitch / 4; g.out_pitch = out_pitch / 4;
    g.kh = kh; g.kw = kw;
    g.kwp = (kw + 3) & ~3;
    g.nw = (g.kwp + 31) / 32;
    g.rw = tile_w + g.kwp + 8;  // the 8-cell chunk loads of the last tap chunk reach tile_w + kwp + 3
    g.tiles_x = (int)((W + tile_w - 1) / tile_w);
    g.n_tiles = (H + 3) / 4 * g.tiles_x;
    return g;
}

// Copies the host table into a buffer ordered on stream s, runs launch_fn(device pointer) and frees the
// buffer after it on the same stream: concurrent calls on distinct streams each use their own copy.
template <typename L>
static int with_device_table(const std::vector<char> &table, cudaStream_t s, L &&launch_fn) {
    void *d = nullptr;
    XRS_CUDA(cudaMallocAsync(&d, table.size(), s));
    const cudaError_t e = cudaMemcpyAsync(d, table.data(), table.size(), cudaMemcpyHostToDevice, s);
    int rc = e == cudaSuccess ? launch_fn(d) : cuda_fail(e, "cudaMemcpyAsync");
    const cudaError_t ef = cudaFreeAsync(d, s);
    if (rc == XRS_OK && ef != cudaSuccess) rc = cuda_fail(ef, "cudaFreeAsync");
    return rc;
}

template <typename... P, typename... A>
static int launch_wide(void (*kern)(P...), const WideGeom &g, cudaStream_t s, LaunchKind kind, const A &...args) {
    const size_t smem = (size_t)kRing * g.rw * sizeof(float);
    int64_t resident;
    if (const int rc = resident_ctas(kern, 256, smem, INT_MAX, &resident)) return rc;
    return launch(kern, resident < g.n_tiles ? resident : g.n_tiles, 256, smem, s, kind, args...);
}

static int conv2d_wide(const float *in, int64_t in_pitch, float *out, int64_t out_pitch, int64_t H, int64_t W,
                       const double *kernel, int kh, int kw, cudaStream_t s) {
    const WideGeom g = wide_geom(in_pitch, out_pitch, H, W, kh, kw, kWideConvW);
    std::vector<char> table((size_t)kh * g.kwp * sizeof(double), 0);  // kh rows of kwp weights, zero padded
    double *w = reinterpret_cast<double *>(table.data());
    for (int ky = 0; ky < kh; ++ky) memcpy(w + (size_t)ky * g.kwp, kernel + (size_t)ky * kw, kw * sizeof(double));
    return with_device_table(table, s, [&](void *d) {
        return launch_wide(conv2d_wide_kernel, g, s, kConvWide, in, (const double *)d, out, g);
    });
}

// Calls f(std::integral_constant<int, S>{}) with S = stat: one xrs_focal_stat, or kAllStats.
template <typename F>
static int with_stat(int stat, F &&f) {
    switch (stat) {
        case XRS_STAT_MEAN: return f(std::integral_constant<int, XRS_STAT_MEAN>{});
        case XRS_STAT_SUM: return f(std::integral_constant<int, XRS_STAT_SUM>{});
        case XRS_STAT_MIN: return f(std::integral_constant<int, XRS_STAT_MIN>{});
        case XRS_STAT_MAX: return f(std::integral_constant<int, XRS_STAT_MAX>{});
        case XRS_STAT_STD: return f(std::integral_constant<int, XRS_STAT_STD>{});
        case XRS_STAT_RANGE: return f(std::integral_constant<int, XRS_STAT_RANGE>{});
        case XRS_STAT_VAR: return f(std::integral_constant<int, XRS_STAT_VAR>{});
        default: return f(std::integral_constant<int, kAllStats>{});
    }
}

// stat: one xrs_focal_stat into planes.p[stat], or kAllStats
static int focal_wide(const float *in, int64_t in_pitch, const StatPlanes &planes, int64_t out_pitch, int64_t H,
                      int64_t W, const double *kernel, int kh, int kw, int stat, cudaStream_t s) {
    const WideGeom g = wide_geom(in_pitch, out_pitch, H, W, kh, kw, kWideStatW);
    // kh spans [lo, hi) (4-tap chunks holding the row's ones; lo = kwp, hi = 0 for a row without any), then
    // kh rows of nw mask words
    const size_t span_bytes = (size_t)kh * sizeof(int2);
    std::vector<char> table(span_bytes + (size_t)kh * g.nw * sizeof(uint32_t), 0);
    int2 *span = reinterpret_cast<int2 *>(table.data());
    uint32_t *bits = reinterpret_cast<uint32_t *>(table.data() + span_bytes);
    for (int ky = 0; ky < kh; ++ky) {
        int first = -1, last = -1;
        for (int kx = 0; kx < kw; ++kx)
            if (kernel[(size_t)ky * kw + kx] == 1.0) {  // focal.py:323
                bits[(size_t)ky * g.nw + kx / 32] |= 1u << (kx % 32);
                if (first < 0) first = kx;
                last = kx;
            }
        span[ky] = first < 0 ? make_int2(g.kwp, 0) : make_int2(first & ~3, (last + 4) & ~3);
    }
    return with_device_table(table, s, [&](void *d) {
        const int2 *dspan = (const int2 *)d;
        const uint32_t *dbits = (const uint32_t *)((const char *)d + span_bytes);
        return with_stat(stat, [&](auto S) {
            return launch_wide(focal_wide_kernel<S>, g, s, S == kAllStats ? kFocalWideFused : kFocalWide, in, dspan,
                               dbits, planes, g);
        });
    });
}

// The tiled and bounds-checked kernels' mask (focal.py:323: the cells where the kernel is 1); returns whether the
// window is all ones.
static bool mask_bits(MaskBits &mask, const double *kernel, int kh, int kw) {
    bool all_ones = true;
    for (int i = 0; i < kh * kw; ++i) {
        mask.m[i] = (kernel[i] == 1.0) ? 1 : 0;
        all_ones = all_ones && mask.m[i];
    }
    return all_ones;
}

static int check_common(const float *in, int64_t in_pitch, float *out, int64_t out_pitch, int64_t H, int64_t W,
                        const double *kernel, int kh, int kw) {
    XRS_REQUIRE(in && out && kernel, "NULL pointer");
    XRS_REQUIRE((const void *)in != (const void *)out, "in and out must not alias");
    if (const int rc = check_window(kh, kw)) return rc;
    XRS_REQUIRE(in_pitch % 4 == 0 && in_pitch >= W * 4 && out_pitch % 4 == 0 && out_pitch >= W * 4,
                "pitches must be multiples of 4 bytes and >= row bytes");
    XRS_REQUIRE(H < (1LL << 31) - 64 && W < (1LL << 31) - 256, "raster dimension too large");
    return XRS_OK;
}

static bool tile_geom(TileGeom &g, CUtensorMap *tmap, const float *in, int64_t in_pitch, float *out,
                      int64_t out_pitch, int64_t H, int64_t W, int kh, int kw, int tile_h) {
    g.H = H; g.W = W; g.kh = kh; g.kw = kw; g.ry = kh / 2; g.rx = kw / 2;
    g.pad = (g.rx + 3) / 4 * 4;
    g.off = g.pad - g.rx;
    // the 8-wide chunk loads of the convolution reach 4*31 + 4*((off+kw-1)/4) + 7 cells into a row
    g.sw = kTileW + ((g.off + kw + 3) / 4) * 4 + 4;
    g.sh = tile_h + kh - 1;
    g.tiles_x = (int)((W + kTileW - 1) / kTileW);
    g.tiles_y = (int)((H + tile_h - 1) / tile_h);
    g.box_h = g.sh <= 64 ? g.sh : 64;  // 64 % 8 == 0 keeps the following boxes 128-byte aligned
    if (g.sw > 256) return false;
    if (W % 4 != 0 || out_pitch % 16 != 0 || (reinterpret_cast<uintptr_t>(out) & 15)) return false;
    return make_tensor_map_2d(tmap, in, in_pitch, H, W, XRS_F32, g.sw, g.box_h) && g.smem_bytes() <= kSmemPerCtaMax;
}

// The persistent tiled kernels: 256 threads, as many CTAs as fit (at most max_per_sm per SM), never more CTAs
// than tiles.
template <typename... P, typename... A>
static int launch_tiles(void (*kern)(P...), const TileGeom &g, int max_per_sm, cudaStream_t s, LaunchKind kind,
                        const A &...args) {
    const size_t smem = g.smem_bytes();
    int64_t resident;
    if (const int rc = resident_ctas(kern, 256, smem, max_per_sm, &resident)) return rc;
    const int64_t n_tiles = (int64_t)g.tiles_x * g.tiles_y;
    return launch(kern, resident < n_tiles ? resident : n_tiles, 256, smem, s, kind, args...);
}

}  // namespace xrs

using namespace xrs;

int xrs_conv3_strip(const float *in, int64_t in_pitch, float *out, int64_t out_pitch, int64_t H, int64_t W,
                    const double *kernel, cudaStream_t s);  // surface.cu
namespace xrs {
// The focal statistics of one raster: stat is one xrs_focal_stat, written to planes.p[stat], or kAllStats for
// every plane that is set.  A wide window takes the ring kernel; a single mean over an all-ones window the running
// box; a raster TMA can describe the tiled kernel, one launch for all the planes; any other raster the
// bounds-checked kernel, one plane at a time.
static int focal_stats(const float *in, int64_t in_pitch, const StatPlanes &planes, int64_t out_pitch, int64_t H,
                       int64_t W, const double *kernel, int kh, int kw, int stat, cudaStream_t s) {
    if (is_wide(kh, kw)) return focal_wide(in, in_pitch, planes, out_pitch, H, W, kernel, kh, kw, stat, s);
    static thread_local MaskBits mask;
    const bool all_ones = mask_bits(mask, kernel, kh, kw);
    int brc;
    if (stat == XRS_STAT_MEAN && all_ones &&   // np.ones((k, k))
        try_running_box(BoxMode::kNanMean, 1.0 / (double)(kh * kw), in, in_pitch, planes.p[stat], out_pitch, H, W, kh,
                        kw, s, &brc))
        return brc;
    float *out = nullptr;  // any plane: the planes share their alignment
    for (float *p : planes.p)
        if (p) out = p;
    TileGeom g;
    CUtensorMap tmap;
    if (tile_geom(g, &tmap, in, in_pitch, out, out_pitch, H, W, kh, kw, kTileH))
        return with_stat(stat, [&](auto S) {
            // at most 3 CTAs per SM (registers differ a lot between the statistics): the tile loop is persistent
            return launch_tiles(focal_tile_kernel<S>, g, 3, s, S == kAllStats ? kFocalFused : kFocalTiled, tmap,
                                mask, focal_out<S>(planes), out_pitch / 4, g);
        });
    const int64_t cell_ctas = (H * W + 255) / 256, max_ctas = (int64_t)sm_count() * 8;
    for (int i = 0; i < 7; ++i) {
        if (!planes.p[i]) continue;
        const int rc = launch(focal_stat_direct_kernel, cell_ctas < max_ctas ? cell_ctas : max_ctas, 256, 0, s,
                              kFocalDirect, in, in_pitch / 4, mask, planes.p[i], out_pitch / 4, H, W, kh, kw, i);
        if (rc) return rc;
    }
    return XRS_OK;
}
}

extern "C" {

int xrs_convolve2d_f32(const float *in, int64_t in_pitch, float *out, int64_t out_pitch, int64_t H, int64_t W,
                       const double *kernel, int kh, int kw, xrs_stream_t s) {
    if (H <= 0 || W <= 0) return XRS_OK;
    const int rc = check_common(in, in_pitch, out, out_pitch, H, W, kernel, kh, kw);
    if (rc) return rc;
    if (is_wide(kh, kw)) return conv2d_wide(in, in_pitch, out, out_pitch, H, W, kernel, kh, kw, (cudaStream_t)s);
    if (kh == 3 && kw == 3) return xrs_conv3_strip(in, in_pitch, out, out_pitch, H, W, kernel, (cudaStream_t)s);
    const double w = kernel[0];   // all taps bitwise equal to a finite w (np.ones((k, k)) / k**2): the running box
    bool uniform = fabs(w) <= 1.7976931348623157e308;
    for (int i = 1; uniform && i < kh * kw; ++i) uniform = memcmp(&kernel[i], &w, sizeof(double)) == 0;
    int brc;
    if (uniform &&
        try_running_box(BoxMode::kConvolve, w, in, in_pitch, out, out_pitch, H, W, kh, kw, (cudaStream_t)s, &brc))
        return brc;
    static thread_local ConvWeights cw;
    for (int i = 0; i < kh * kw; ++i) cw.w[i] = kernel[i];
    TileGeom g;
    CUtensorMap tmap;
    if (tile_geom(g, &tmap, in, in_pitch, out, out_pitch, H, W, kh, kw, kConvTileH)) {
        auto kern = conv2d_kernel<0>;
        if (kh == kw && kw >= 5 && kw <= 13) {
            switch (kw) {
                case 5: kern = conv2d_fixed_kernel<5>; break;
                case 7: kern = conv2d_fixed_kernel<7>; break;
                case 11: kern = conv2d_fixed_kernel<11>; break;
                case 13: kern = conv2d_fixed_kernel<13>; break;
                default: kern = conv2d_fixed_kernel<9>; break;
            }
        } else {
            switch (kw) {
                case 5: kern = conv2d_kernel<5>; break;
                case 7: kern = conv2d_kernel<7>; break;
                case 9: kern = conv2d_kernel<9>; break;
            }
        }
        return launch_tiles(kern, g, INT_MAX, (cudaStream_t)s, kConvTiled, tmap, cw, out, out_pitch / 4, g);
    }
    const int64_t cell_ctas = (H * W + 255) / 256, max_ctas = (int64_t)sm_count() * 8;
    return launch(conv2d_direct_kernel, cell_ctas < max_ctas ? cell_ctas : max_ctas, 256, 0, (cudaStream_t)s,
                  kConvDirect, in, in_pitch / 4, cw, out, out_pitch / 4, H, W, kh, kw);
}

int xrs_focal_stat_f32(const float *in, int64_t in_pitch, float *out, int64_t out_pitch, int64_t H, int64_t W,
                       const double *kernel, int kh, int kw, int stat, xrs_stream_t s) {
    if (H <= 0 || W <= 0) return XRS_OK;
    const int rc = check_common(in, in_pitch, out, out_pitch, H, W, kernel, kh, kw);
    if (rc) return rc;
    XRS_REQUIRE(stat >= XRS_STAT_MEAN && stat <= XRS_STAT_VAR, "unknown focal statistic");
    StatPlanes planes = {};
    planes.p[stat] = out;
    return focal_stats(in, in_pitch, planes, out_pitch, H, W, kernel, kh, kw, stat, (cudaStream_t)s);
}

int xrs_focal_stats_multi_f32(const float *in, int64_t in_pitch, float *out, int64_t out_pitch, int64_t plane_stride,
                              int64_t H, int64_t W, const double *kernel, int kh, int kw, const int *stats,
                              int n_stats, xrs_stream_t s) {
    XRS_REQUIRE(stats != nullptr && n_stats >= 1 && n_stats <= 7, "stats: 1..7 statistic ids");
    XRS_REQUIRE(plane_stride % 16 == 0 && plane_stride >= H * out_pitch, "plane_stride must cover one plane (16-byte multiple)");
    if (H <= 0 || W <= 0) return XRS_OK;
    const int rc = check_common(in, in_pitch, out, out_pitch, H, W, kernel, kh, kw);
    if (rc) return rc;
    StatPlanes planes = {};
    for (int i = 0; i < n_stats; ++i) {
        XRS_REQUIRE(stats[i] >= XRS_STAT_MEAN && stats[i] <= XRS_STAT_VAR, "unknown focal statistic");
        XRS_REQUIRE(planes.p[stats[i]] == nullptr, "statistic requested twice");
        planes.p[stats[i]] = reinterpret_cast<float *>(reinterpret_cast<char *>(out) + (int64_t)i * plane_stride);
    }
    // one statistic takes its own kernels
    return focal_stats(in, in_pitch, planes, out_pitch, H, W, kernel, kh, kw, n_stats == 1 ? stats[0] : kAllStats,
                       (cudaStream_t)s);
}

}  // extern "C"

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
};

__device__ __forceinline__ void load_tile_tma(const CUtensorMap *tmap, float *tile32, uint64_t *bar,
                                              const TileGeom &g, int tx0, int ty0, uint32_t parity) {
    // one elected thread issues the boxes; everyone waits on the mbarrier
    if (threadIdx.x == 0) {
        const int nbox = (g.sh + g.box_h - 1) / g.box_h;
        mbar_arrive_expect_tx(bar, (uint32_t)(nbox * g.box_h * g.sw * sizeof(float)));
        for (int b = 0; b < nbox; ++b)
            tma_load_2d(tile32 + (size_t)b * g.box_h * g.sw, tmap, bar, tx0 - g.pad, ty0 - g.ry + b * g.box_h);
    }
    mbar_wait(bar, parity);
}

// ----------------------------------------------------------------------------- convolve
// 128 x 64 output tile per CTA, 256 threads = 16 (x) x 16 (y); a thread owns 4 rows x (4 + 4)
// columns: columns 4tx .. 4tx+3 and 64+4tx .. 64+4tx+3, so that consecutive lanes read
// consecutive 16-byte pieces of a shared-memory row (conflict-free LDS.128).  The float32 tile
// is read directly and widened in registers (16 F2F per 128 DFMA); 32 independent float64
// accumulators per thread give the FP64 pipe enough parallelism at 2-3 CTAs per SM.
constexpr int kConvTileH = 64;

// KW > 0: kernel width known at compile time (5, 7, 9: the usual custom kernels) -- the tap-chunk
// loop unrolls and its chunk / tap tests fold away; KW == 0: any odd shape.
template <int KW>
__global__ void __launch_bounds__(256)
conv2d_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ ConvWeights cw,
              float *__restrict__ out, int64_t out_pitch_elems, const TileGeom g) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    const int nbox = (g.sh + g.box_h - 1) / g.box_h;
    const size_t tile_cells = (size_t)nbox * g.box_h * g.sw;
    float *tile32 = reinterpret_cast<float *>(smem_raw);
    uint64_t *bar = reinterpret_cast<uint64_t *>(smem_raw + tile_cells * sizeof(float));

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmap);
        mbar_init(bar, 1);
        mbar_fence_init();
    }
    __syncthreads();

    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int64_t n_tiles = (int64_t)g.tiles_x * g.tiles_y;
    uint32_t parity = 0;
    for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const int tile_y = (int)(t / g.tiles_x), tile_x = (int)(t % g.tiles_x);
        const int x0 = tile_x * kTileW, y0 = tile_y * kConvTileH;
        load_tile_tma(&tmap, tile32, bar, g, x0, y0, parity);
        parity ^= 1u;

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
        const int64_t xa = (int64_t)x0 + 4 * tx, xb = xa + 64;
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int64_t yo = (int64_t)y0 + ty * 4 + r;
            if (yo < g.H) {  // W % 4 == 0 on this path: a float4 is all-in or all-out
                float *orow = out + yo * out_pitch_elems;
                if (xa < g.W)
                    __stcs(reinterpret_cast<float4 *>(orow + xa),
                           make_float4((float)acc[r][0], (float)acc[r][1], (float)acc[r][2], (float)acc[r][3]));
                if (xb < g.W)
                    __stcs(reinterpret_cast<float4 *>(orow + xb),
                           make_float4((float)acc[r][4], (float)acc[r][5], (float)acc[r][6], (float)acc[r][7]));
            }
        }
        __syncthreads();  // the tile buffer is reused by the next iteration
    }
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
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    const int nbox = (g.sh + g.box_h - 1) / g.box_h;
    const size_t tile_cells = (size_t)nbox * g.box_h * g.sw;
    float *tile32 = reinterpret_cast<float *>(smem_raw);
    uint64_t *bar = reinterpret_cast<uint64_t *>(smem_raw + tile_cells * sizeof(float));
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmap);
        mbar_init(bar, 1);
        mbar_fence_init();
    }
    __syncthreads();
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int64_t n_tiles = (int64_t)g.tiles_x * g.tiles_y;
    uint32_t parity = 0;
    for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const int tile_y = (int)(t / g.tiles_x), tile_x = (int)(t % g.tiles_x);
        const int x0 = tile_x * kTileW, y0 = tile_y * kConvTileH;
        load_tile_tma(&tmap, tile32, bar, g, x0, y0, parity);
        parity ^= 1u;
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
        const int64_t xa = (int64_t)x0 + 4 * tx, xb = xa + 64;
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int64_t yo = (int64_t)y0 + ty * 4 + r;
            if (yo < g.H) {
                float *orow = out + yo * out_pitch_elems;
                if (xa < g.W)
                    __stcs(reinterpret_cast<float4 *>(orow + xa),
                           make_float4((float)acc[r][0], (float)acc[r][1], (float)acc[r][2], (float)acc[r][3]));
                if (xb < g.W)
                    __stcs(reinterpret_cast<float4 *>(orow + xb),
                           make_float4((float)acc[r][4], (float)acc[r][5], (float)acc[r][6], (float)acc[r][7]));
            }
        }
        __syncthreads();
    }
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

// Register-blocked like conv2d_kernel: a thread owns 4 x 4 outputs, walks the input rows of its
// window once (twice for var / std), loads 8 cells per 4-tap chunk with two LDS.128 and feeds
// every (output row, tap) pair whose mask bit is set.  Taps are visited in row-major window
// order for each output, so the float32 `sum` is bit-identical to np.nansum on the scratch.
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

template <typename F>
__device__ __forceinline__ void focal_sweep(const float *tile32, const MaskBits &mask, const TileGeom &g, int tx,
                                            int ty, F &&f) {
    const int rows_in = 4 + g.kh - 1;
    const int n_taps = g.off + g.kw;
    for (int j = 0; j < rows_in; ++j) {
        const float *rowp = tile32 + (size_t)(ty * 4 + j) * g.sw + 4 * tx;
        for (int kb = 0; kb < n_taps; kb += 4) {
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

template <int STAT>
__global__ void __launch_bounds__(256)
focal_stat_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ MaskBits mask,
                  float *__restrict__ out, int64_t out_pitch_elems, const TileGeom g) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    const int nbox = (g.sh + g.box_h - 1) / g.box_h;
    const size_t tile_cells = (size_t)nbox * g.box_h * g.sw;
    float *tile32 = reinterpret_cast<float *>(smem_raw);
    uint64_t *bar = reinterpret_cast<uint64_t *>(smem_raw + tile_cells * sizeof(float));
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmap);
        mbar_init(bar, 1);
        mbar_fence_init();
    }
    __syncthreads();
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int64_t n_tiles = (int64_t)g.tiles_x * g.tiles_y;
    uint32_t parity = 0;
    for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const int tile_y = (int)(t / g.tiles_x), tile_x = (int)(t % g.tiles_x);
        const int x0 = tile_x * kTileW, y0 = tile_y * kTileH;
        load_tile_tma(&tmap, tile32, bar, g, x0, y0, parity);
        parity ^= 1u;
        float res[4][4];
        if constexpr (STAT == XRS_STAT_MEAN || STAT == XRS_STAT_VAR || STAT == XRS_STAT_STD) {
            double sum[4][4];
            int cnt[4][4];
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c) sum[r][c] = 0.0, cnt[r][c] = 0;
            focal_sweep(tile32, mask, g, tx, ty, [&](int r, int c, const FocalCell &q) {
                sum[r][c] += q.dz;
                cnt[r][c] += q.one;
            });
            if constexpr (STAT == XRS_STAT_MEAN) {
#pragma unroll
                for (int r = 0; r < 4; ++r)
#pragma unroll
                    for (int c = 0; c < 4; ++c) res[r][c] = (float)(sum[r][c] / (double)cnt[r][c]);
            } else {
                double ssd[4][4];
#pragma unroll
                for (int r = 0; r < 4; ++r)
#pragma unroll
                    for (int c = 0; c < 4; ++c) sum[r][c] = sum[r][c] / (double)cnt[r][c], ssd[r][c] = 0.0;
                focal_sweep(tile32, mask, g, tx, ty, [&](int r, int c, const FocalCell &q) {
                    const double d = q.d - sum[r][c];
                    ssd[r][c] += q.ok ? d * d : 0.0;
                });
#pragma unroll
                for (int r = 0; r < 4; ++r)
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        const double var = ssd[r][c] / (double)cnt[r][c];
                        res[r][c] = (float)(STAT == XRS_STAT_VAR ? var : sqrt(var));
                    }
            }
        } else if constexpr (STAT == XRS_STAT_SUM) {
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c) res[r][c] = 0.f;
            focal_sweep(tile32, mask, g, tx, ty, [&](int r, int c, const FocalCell &q) { res[r][c] += q.vz; });
        } else {
            float mn[4][4], mx[4][4];
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c) mn[r][c] = mx[r][c] = nan_of<float>();
            focal_sweep(tile32, mask, g, tx, ty, [&](int r, int c, const FocalCell &q) {
                nan_min_step(mn[r][c], q.v);
                nan_max_step(mx[r][c], q.v);
            });
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c)
                    res[r][c] = STAT == XRS_STAT_MIN ? mn[r][c] : STAT == XRS_STAT_MAX ? mx[r][c] : mx[r][c] - mn[r][c];
        }
        const int64_t xo = (int64_t)x0 + 4 * tx;
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int64_t yo = (int64_t)y0 + ty * 4 + r;
            if (yo < g.H && xo < g.W)  // W % 4 == 0 on this path
                __stcs(reinterpret_cast<float4 *>(out + yo * out_pitch_elems + xo),
                       make_float4(res[r][0], res[r][1], res[r][2], res[r][3]));
        }
        __syncthreads();
    }
}

// All requested statistics of one window in ONE pass over the raster (focal.focal_stats,
// focal.py:800-878, is seven `apply` calls stacked with xr.concat): the tile is loaded once,
// sweep A accumulates the float64 sum, the count and the float32 row-major sum of every output's
// window, sweep B the min / max and the squared deviations about the float64 mean, and each
// statistic goes straight into its plane of the (stats, y, x) result -- 2 sweeps and one tile
// load instead of 9 and 7, and no stacking copy.  Per-statistic arithmetic is the single-stat
// kernel's, operation for operation.
struct StatPlanes {
    float *p[7];  // indexed by xrs_focal_stat; nullptr = not requested
};

__device__ __forceinline__ void store_tile16(float *plane, int64_t pitch_elems, int64_t H, int64_t W, int64_t y0,
                                             int64_t xo, const float (&res)[4][4]) {
#pragma unroll
    for (int r = 0; r < 4; ++r)
        if (y0 + r < H && xo < W)  // W % 4 == 0 on this path
            __stcs(reinterpret_cast<float4 *>(plane + (y0 + r) * pitch_elems + xo),
                   make_float4(res[r][0], res[r][1], res[r][2], res[r][3]));
}

__global__ void __launch_bounds__(256, 2)
focal_stats_multi_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ MaskBits mask,
                         const StatPlanes planes, int64_t out_pitch_elems, const TileGeom g) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    const int nbox = (g.sh + g.box_h - 1) / g.box_h;
    const size_t tile_cells = (size_t)nbox * g.box_h * g.sw;
    float *tile32 = reinterpret_cast<float *>(smem_raw);
    uint64_t *bar = reinterpret_cast<uint64_t *>(smem_raw + tile_cells * sizeof(float));
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmap);
        mbar_init(bar, 1);
        mbar_fence_init();
    }
    __syncthreads();
    const bool want_b = planes.p[XRS_STAT_MIN] || planes.p[XRS_STAT_MAX] || planes.p[XRS_STAT_RANGE] ||
                        planes.p[XRS_STAT_STD] || planes.p[XRS_STAT_VAR];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int64_t n_tiles = (int64_t)g.tiles_x * g.tiles_y;
    uint32_t parity = 0;
    for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const int tile_y = (int)(t / g.tiles_x), tile_x = (int)(t % g.tiles_x);
        const int x0 = tile_x * kTileW, y0 = tile_y * kTileH;
        load_tile_tma(&tmap, tile32, bar, g, x0, y0, parity);
        parity ^= 1u;
        const int64_t xo = (int64_t)x0 + 4 * tx, yo = (int64_t)y0 + ty * 4;
        float res[4][4];
        double mean[4][4];
        int cnt[4][4];
        {
            float fsum[4][4];
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c) mean[r][c] = 0.0, cnt[r][c] = 0, fsum[r][c] = 0.f;
            focal_sweep(tile32, mask, g, tx, ty, [&](int r, int c, const FocalCell &q) {
                mean[r][c] += q.dz;
                cnt[r][c] += q.one;
                fsum[r][c] += q.vz;
            });
            if (planes.p[XRS_STAT_SUM]) store_tile16(planes.p[XRS_STAT_SUM], out_pitch_elems, g.H, g.W, yo, xo, fsum);
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    mean[r][c] = mean[r][c] / (double)cnt[r][c];
                    res[r][c] = (float)mean[r][c];
                }
            if (planes.p[XRS_STAT_MEAN]) store_tile16(planes.p[XRS_STAT_MEAN], out_pitch_elems, g.H, g.W, yo, xo, res);
        }
        if (want_b) {
            float mn[4][4], mx[4][4];
            double ssd[4][4];
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c) mn[r][c] = mx[r][c] = nan_of<float>(), ssd[r][c] = 0.0;
            focal_sweep(tile32, mask, g, tx, ty, [&](int r, int c, const FocalCell &q) {
                const double d = q.d - mean[r][c];
                ssd[r][c] += q.ok ? d * d : 0.0;
                nan_min_step(mn[r][c], q.v);
                nan_max_step(mx[r][c], q.v);
            });
            if (planes.p[XRS_STAT_MIN]) store_tile16(planes.p[XRS_STAT_MIN], out_pitch_elems, g.H, g.W, yo, xo, mn);
            if (planes.p[XRS_STAT_MAX]) store_tile16(planes.p[XRS_STAT_MAX], out_pitch_elems, g.H, g.W, yo, xo, mx);
            if (planes.p[XRS_STAT_RANGE]) {
#pragma unroll
                for (int r = 0; r < 4; ++r)
#pragma unroll
                    for (int c = 0; c < 4; ++c) res[r][c] = mx[r][c] - mn[r][c];
                store_tile16(planes.p[XRS_STAT_RANGE], out_pitch_elems, g.H, g.W, yo, xo, res);
            }
            if (planes.p[XRS_STAT_VAR] || planes.p[XRS_STAT_STD]) {
#pragma unroll
                for (int r = 0; r < 4; ++r)
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        ssd[r][c] = ssd[r][c] / (double)cnt[r][c];
                        res[r][c] = (float)ssd[r][c];
                    }
                if (planes.p[XRS_STAT_VAR]) store_tile16(planes.p[XRS_STAT_VAR], out_pitch_elems, g.H, g.W, yo, xo, res);
                if (planes.p[XRS_STAT_STD]) {
#pragma unroll
                    for (int r = 0; r < 4; ++r)
#pragma unroll
                        for (int c = 0; c < 4; ++c) res[r][c] = (float)sqrt(ssd[r][c]);
                    store_tile16(planes.p[XRS_STAT_STD], out_pitch_elems, g.H, g.W, yo, xo, res);
                }
            }
        }
        __syncthreads();
    }
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

static int check_common(const float *in, int64_t in_pitch, float *out, int64_t out_pitch, int64_t H, int64_t W,
                        const double *kernel, int kh, int kw) {
    XRS_REQUIRE(in && out && kernel, "NULL pointer");
    XRS_REQUIRE((const void *)in != (const void *)out, "in and out must not alias");
    XRS_REQUIRE(kh >= 1 && kw >= 1 && (kh & 1) && (kw & 1), "kernel dimensions must be odd");
    XRS_REQUIRE(kh * kw <= kMaxTaps && kh <= 63 && kw <= 63, "kernel too large (max 49x49 taps, 63 per side)");
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
    return make_tensor_map_2d(tmap, in, in_pitch, H, W, 4, g.sw, g.box_h);
}

}  // namespace xrs

using namespace xrs;

int xrs_conv3_strip(const float *in, int64_t in_pitch, float *out, int64_t out_pitch, int64_t H, int64_t W,
                    const double *kernel, cudaStream_t s);  // surface.cu
namespace xrs {
bool try_box_stream(const float *in, int64_t in_pitch, float *out, int64_t out_pitch, int64_t H, int64_t W,
                    const double *kernel, int kh, int kw, cudaStream_t s, int *rc);
// box_stream.cu, NaN-skipping mode: focal.apply mean over an all-ones window
bool try_box_nanmean(const float *in, int64_t in_pitch, float *out, int64_t out_pitch, int64_t H, int64_t W,
                     int kh, int kw, cudaStream_t s, int *rc);  // box_stream.cu
}

extern "C" {

int xrs_convolve2d_f32(const float *in, int64_t in_pitch, float *out, int64_t out_pitch, int64_t H, int64_t W,
                       const double *kernel, int kh, int kw, xrs_stream_t s) {
    if (H <= 0 || W <= 0) return XRS_OK;
    const int rc = check_common(in, in_pitch, out, out_pitch, H, W, kernel, kh, kw);
    if (rc) return rc;
    if (kh == 3 && kw == 3) return xrs_conv3_strip(in, in_pitch, out, out_pitch, H, W, kernel, (cudaStream_t)s);
    {
        int brc = XRS_OK;
        // all taps bitwise equal, k <= 25 per side, TMA-describable raster: streaming running-box kernel
        if (try_box_stream(in, in_pitch, out, out_pitch, H, W, kernel, kh, kw, (cudaStream_t)s, &brc)) return brc;
    }
    static thread_local ConvWeights cw;
    for (int i = 0; i < kh * kw; ++i) cw.w[i] = kernel[i];
    TileGeom g;
    CUtensorMap tmap;
    const int sms = sm_count();
    if (tile_geom(g, &tmap, in, in_pitch, out, out_pitch, H, W, kh, kw, kConvTileH)) {
        const int nbox = (g.sh + g.box_h - 1) / g.box_h;
        const size_t cells = (size_t)nbox * g.box_h * g.sw;
        const size_t smem = cells * 4 + 16;
        if (smem <= 227 * 1024) {
            const int64_t n_tiles = (int64_t)g.tiles_x * g.tiles_y;
            int64_t grid = 0;
#define XRS_CONV(KWC)                                                                                          \
    {                                                                                                          \
        XRS_CUDA(cudaFuncSetAttribute(conv2d_kernel<KWC>, cudaFuncAttributeMaxDynamicSharedMemorySize,        \
                                      (int)smem));                                                             \
        int per_sm = 0;                                                                                        \
        XRS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, conv2d_kernel<KWC>, 256, smem));      \
        if (per_sm < 1) per_sm = 1;                                                                            \
        grid = (int64_t)sms * per_sm;                                                                          \
        if (grid > n_tiles) grid = n_tiles;                                                                    \
        conv2d_kernel<KWC><<<(unsigned)grid, 256, smem, (cudaStream_t)s>>>(tmap, cw, out, out_pitch / 4, g);  \
    }
#define XRS_CONVF(KC)                                                                                           \
    {                                                                                                          \
        XRS_CUDA(cudaFuncSetAttribute(conv2d_fixed_kernel<KC>, cudaFuncAttributeMaxDynamicSharedMemorySize,   \
                                      (int)smem));                                                             \
        int per_sm = 0;                                                                                        \
        XRS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, conv2d_fixed_kernel<KC>, 256, smem)); \
        if (per_sm < 1) per_sm = 1;                                                                            \
        grid = (int64_t)sms * per_sm;                                                                          \
        if (grid > n_tiles) grid = n_tiles;                                                                    \
        conv2d_fixed_kernel<KC><<<(unsigned)grid, 256, smem, (cudaStream_t)s>>>(tmap, cw, out, out_pitch / 4, g); \
    }
            if (kh == kw && kw >= 5 && kw <= 13) {
                switch (kw) {
                    case 5: XRS_CONVF(5) break;
                    case 7: XRS_CONVF(7) break;
                    case 11: XRS_CONVF(11) break;
                    case 13: XRS_CONVF(13) break;
                    default: XRS_CONVF(9) break;
                }
            } else
            switch (kw) {
                case 5: XRS_CONV(5) break;
                case 7: XRS_CONV(7) break;
                case 9: XRS_CONV(9) break;
                default: XRS_CONV(0) break;
            }
#undef XRS_CONV
#undef XRS_CONVF
            XRS_CUDA(cudaGetLastError());
            last_launch_info() = {4, (int)grid, 256, (int)smem};
            return XRS_OK;
        }
    }
    int64_t grid = (H * W + 255) / 256;
    if (grid > (int64_t)sms * 8) grid = (int64_t)sms * 8;
    conv2d_direct_kernel<<<(unsigned)grid, 256, 0, (cudaStream_t)s>>>(in, in_pitch / 4, cw, out, out_pitch / 4, H, W,
                                                                     kh, kw);
    last_launch_info() = {5, (int)grid, 256, 0};
    XRS_CUDA(cudaGetLastError());
    return XRS_OK;
}

int xrs_focal_stat_f32(const float *in, int64_t in_pitch, float *out, int64_t out_pitch, int64_t H, int64_t W,
                       const double *kernel, int kh, int kw, int stat, xrs_stream_t s) {
    if (H <= 0 || W <= 0) return XRS_OK;
    const int rc = check_common(in, in_pitch, out, out_pitch, H, W, kernel, kh, kw);
    if (rc) return rc;
    XRS_REQUIRE(stat >= XRS_STAT_MEAN && stat <= XRS_STAT_VAR, "unknown focal statistic");
    static thread_local MaskBits mask;
    bool all_ones = true;
    for (int i = 0; i < kh * kw; ++i) {
        mask.m[i] = (kernel[i] == 1.0) ? 1 : 0;  // focal.py:323
        all_ones = all_ones && mask.m[i];
    }
    if (stat == XRS_STAT_MEAN && all_ones) {   // np.ones((k, k)): the running box, O(1) per cell
        int brc = XRS_OK;
        if (try_box_nanmean(in, in_pitch, out, out_pitch, H, W, kh, kw, (cudaStream_t)s, &brc)) return brc;
    }
    TileGeom g;
    CUtensorMap tmap;
    const int sms = sm_count();
    if (tile_geom(g, &tmap, in, in_pitch, out, out_pitch, H, W, kh, kw, kTileH)) {
        const int nbox = (g.sh + g.box_h - 1) / g.box_h;
        const size_t smem = (size_t)nbox * g.box_h * g.sw * 4 + 16;
        if (smem <= 227 * 1024) {
            const int64_t n_tiles = (int64_t)g.tiles_x * g.tiles_y;
            int64_t grid = 0;
            // resident CTAs only (registers differ a lot between the statistics): the tile loop is persistent
#define XRS_FS(ST)                                                                                              \
    case ST: {                                                                                                  \
        XRS_CUDA(cudaFuncSetAttribute(focal_stat_kernel<ST>, cudaFuncAttributeMaxDynamicSharedMemorySize,     \
                                      (int)smem));                                                              \
        int per_sm = 0;                                                                                         \
        XRS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, focal_stat_kernel<ST>, 256, smem));    \
        per_sm = per_sm < 1 ? 1 : (per_sm > 3 ? 3 : per_sm);                                                    \
        grid = (int64_t)sms * per_sm;                                                                           \
        if (grid > n_tiles) grid = n_tiles;                                                                     \
        focal_stat_kernel<ST><<<(unsigned)grid, 256, smem, (cudaStream_t)s>>>(tmap, mask, out, out_pitch / 4, g); \
        break;                                                                                                  \
    }
            switch (stat) {
                XRS_FS(XRS_STAT_MEAN) XRS_FS(XRS_STAT_SUM) XRS_FS(XRS_STAT_MIN) XRS_FS(XRS_STAT_MAX)
                XRS_FS(XRS_STAT_STD) XRS_FS(XRS_STAT_RANGE) XRS_FS(XRS_STAT_VAR)
            }
#undef XRS_FS
            XRS_CUDA(cudaGetLastError());
            last_launch_info() = {7, (int)grid, 256, (int)smem};
            return XRS_OK;
        }
    }
    int64_t grid = (H * W + 255) / 256;
    if (grid > (int64_t)sms * 8) grid = (int64_t)sms * 8;
    focal_stat_direct_kernel<<<(unsigned)grid, 256, 0, (cudaStream_t)s>>>(in, in_pitch / 4, mask, out, out_pitch / 4,
                                                                         H, W, kh, kw, stat);
    last_launch_info() = {8, (int)grid, 256, 0};
    XRS_CUDA(cudaGetLastError());
    return XRS_OK;
}

int xrs_focal_stats_multi_f32(const float *in, int64_t in_pitch, float *out, int64_t out_pitch, int64_t plane_stride,
                              int64_t H, int64_t W, const double *kernel, int kh, int kw, const int *stats,
                              int n_stats, xrs_stream_t s) {
    XRS_REQUIRE(stats != nullptr && n_stats >= 1 && n_stats <= 7, "stats: 1..7 statistic ids");
    XRS_REQUIRE(plane_stride % 16 == 0 && plane_stride >= H * out_pitch, "plane_stride must cover one plane (16-byte multiple)");
    if (H <= 0 || W <= 0) return XRS_OK;
    const int rc = check_common(in, in_pitch, out, out_pitch, H, W, kernel, kh, kw);
    if (rc) return rc;
    StatPlanes planes;
    for (auto &p : planes.p) p = nullptr;
    for (int i = 0; i < n_stats; ++i) {
        XRS_REQUIRE(stats[i] >= XRS_STAT_MEAN && stats[i] <= XRS_STAT_VAR, "unknown focal statistic");
        XRS_REQUIRE(planes.p[stats[i]] == nullptr, "statistic requested twice");
        planes.p[stats[i]] = reinterpret_cast<float *>(reinterpret_cast<char *>(out) + (int64_t)i * plane_stride);
    }
    TileGeom g;
    CUtensorMap tmap;
    if (n_stats >= 2 && tile_geom(g, &tmap, in, in_pitch, out, out_pitch, H, W, kh, kw, kTileH)) {
        const int nbox = (g.sh + g.box_h - 1) / g.box_h;
        const size_t smem = (size_t)nbox * g.box_h * g.sw * 4 + 16;
        if (smem <= 227 * 1024) {
            static thread_local MaskBits mask;
            for (int i = 0; i < kh * kw; ++i) mask.m[i] = (kernel[i] == 1.0) ? 1 : 0;  // focal.py:323
            XRS_CUDA(cudaFuncSetAttribute(focal_stats_multi_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)smem));
            int per_sm = 0;
            XRS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, focal_stats_multi_kernel, 256, smem));
            if (per_sm < 1) per_sm = 1;
            if (per_sm > 3) per_sm = 3;
            int64_t grid = (int64_t)sm_count() * per_sm;
            const int64_t n_tiles = (int64_t)g.tiles_x * g.tiles_y;
            if (grid > n_tiles) grid = n_tiles;
            focal_stats_multi_kernel<<<(unsigned)grid, 256, smem, (cudaStream_t)s>>>(tmap, mask, planes, out_pitch / 4, g);
            XRS_CUDA(cudaGetLastError());
            last_launch_info() = {6, (int)grid, 256, (int)smem};
            return XRS_OK;
        }
    }
    // single statistic, or a raster TMA cannot describe: one launch per plane
    for (int i = 0; i < n_stats; ++i) {
        const int r2 = xrs_focal_stat_f32(in, in_pitch, planes.p[stats[i]], out_pitch, H, W, kernel, kh, kw, stats[i], s);
        if (r2) return r2;
    }
    return XRS_OK;
}

}  // extern "C"

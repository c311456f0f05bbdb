// box_stream.cu -- convolve_2d with a kernel whose taps are all the same weight w
// (np.ones((k, k)) / k**2: the mean filter of the reference's docs and of benchmarks/; also any
// rectangular kh x kw): out = w * (sum of the window), reference convolution.py:285-313.  The same kernel body
// serves focal.apply's mean over an all-ones window (BoxNanMean below, focal.py:305-326).
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
constexpr int kBoxRows = 4;      // rows per stage half (entering / leaving)

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

template <int RX, int NW> struct BoxShape {
    static constexpr int kPad = (RX + 3) / 4 * 4;               // columns a warp cannot emit on each side
    static constexpr int kOutW = kStripW - 2 * kPad;            // columns a warp emits
    static constexpr int kTileOutW = NW * kOutW;
    static constexpr int kTileInW = kTileOutW + 2 * kPad;
    static constexpr int kNBox = (kTileInW + 255) / 256;
    static constexpr int kBoxW = ((kTileInW + kNBox - 1) / kNBox + 31) / 32 * 32;   // cells: 128-byte multiples
    static constexpr int kBoxCells = kBoxRows * kBoxW;          // one TMA box: 4 rows x kBoxW cells
    static constexpr int kHalfCells = kNBox * kBoxCells;        // the entering (or leaving) rows of a stage
    static constexpr uint32_t kHalfBytes = kHalfCells * 4;
    static_assert(kBoxW <= 256 && kBoxW % 32 == 0 && kNBox * kBoxW >= kTileInW, "TMA box geometry");
};

struct BoxGeom {
    int64_t H, W;
    int kh, ry;
    int n_tiles, n_segs, seg_rows;
    int stages;
    double w;        // convolve: the taps' common weight; mean: 1 / (kh * kw)
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

// The kernel's two modes: which loaded cells read as 0, how a window sum becomes the float32 output and how a window
// holding NaN / inf / huge cells is finished.  Built per task for the lane whose first cell is raster column x.

// convolve_2d: out = w * (sum of the window).  A NaN anywhere in the window makes the result NaN, so the columns
// beyond the raster's left / right edge (NaN from the TMA unit) need no masking: they poison exactly their own lane's
// sums, and the windows that contain them come out NaN like the reference's.
template <int RX> struct BoxConvolve {
    __device__ __forceinline__ BoxConvolve(const BoxGeom &, int64_t, bool) {}
    // whether the lane's cells read as 0 in the fast path (FAST) or in the row-by-row path
    template <bool FAST> __device__ __forceinline__ bool zeroes() const { return false; }
    static constexpr bool edge_warp = false;
    // the output of column j's window sum; EDGE: in a warp at the raster's left / right edge
    template <bool EDGE> __device__ __forceinline__ float out(const BoxGeom &g, double win, int) const {
        return (float)fma(g.w, win, 0.0);   // + 0.0: an all-zero window is +0 like the reference's
    }
    // res of column j, whose window holds NaN cells (the low 16 bits of n) or infinite / huge ones (the high 16 bits);
    // `direct`: the lane stores, so the window may be recomputed from `in`
    __device__ __forceinline__ void finish_exceptional(float &res, int j, double win, unsigned n, bool direct,
                                                       const float *in, int64_t pitch, const BoxGeom &g, int64_t y,
                                                       int64_t x) const {
        if (n & 0xffffu) res = nan_of<float>();
        else if ((n >> 16) && direct) res = bs_direct(in, pitch, g.H, g.W, y, x + j, g.kh, 2 * RX + 1, g.w);
    }
};

// focal.apply's mean over an all-ones window: NaN cells and cells beyond the raster are skipped.  Out-of-raster lanes
// read as 0, and a window that reaches over the raster's left / right edge divides by kh x the columns it really has
// (ncv): edge tiles stay on the fast path.
template <int RX> struct BoxNanMean {
    int ncv[4];       // raster columns in the windows of the lane's 4 columns
    bool edge_warp;   // warp-uniform: a window of the warp reaches beyond the raster's left / right edge
    bool outside;     // the lane's cells lie beyond the raster
    __device__ __forceinline__ BoxNanMean(const BoxGeom &g, int64_t x, bool in_raster) : outside(!in_raster) {
        bool edge_lane = false;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int64_t xc = x + j;
            const int64_t lo = xc - RX < 0 ? 0 : xc - RX, hi = xc + RX > g.W - 1 ? g.W - 1 : xc + RX;
            ncv[j] = (int)(hi - lo + 1);
            edge_lane = edge_lane || (ncv[j] != 2 * RX + 1);
        }
        edge_warp = __any_sync(0xffffffffu, edge_lane && in_raster);
    }
    // the fast path tests only the warps at the raster's edges, the only ones whose outputs read such lanes (a warp-
    // uniform branch); the row-by-row path zeroes every out-of-raster lane
    template <bool FAST> __device__ __forceinline__ bool zeroes() const { return FAST ? edge_warp && outside : outside; }
    template <bool EDGE> __device__ __forceinline__ float out(const BoxGeom &g, double win, int j) const {
        return EDGE ? (float)(win / (double)(g.kh * ncv[j])) : (float)bs_div_n(win, g.n_cells, g.w);
    }
    __device__ __forceinline__ void finish_exceptional(float &res, int j, double win, unsigned n, bool direct,
                                                       const float *in, int64_t pitch, const BoxGeom &g, int64_t y,
                                                       int64_t x) const {
        if (n >> 16) {   // infinite / huge cells take part: the reference's order
            if (direct) res = bs_direct_nanmean(in, pitch, g.H, g.W, y, x + j, g.kh, 2 * RX + 1);
        } else if (n & 0xffffu) {
            res = (float)(win / (double)(g.kh * ncv[j] - (int)(n & 0xffffu)));   // all skipped: 0 / 0 = NaN
        }
    }
};

// the lane's 4 cells of one stage row, in the fast path (FAST) or the row-by-row path; the lanes the mode zeroes read 0
template <bool FAST, typename M> __device__ __forceinline__ void bs_row(const M &m, const float *p, float (&v)[4]) {
    const float4 q = *reinterpret_cast<const float4 *>(p);
    v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
    if (m.template zeroes<FAST>()) { v[0] = 0.f; v[1] = 0.f; v[2] = 0.f; v[3] = 0.f; }
}

// the lane's 4 outputs of one row
template <bool EDGE, typename M>
__device__ __forceinline__ void bs_store(const M &m, float *p, const BoxGeom &g, const double (&win)[4]) {
    __stcs(reinterpret_cast<float4 *>(p), make_float4(m.template out<EDGE>(g, win[0], 0), m.template out<EDGE>(g, win[1], 1),
                                                      m.template out<EDGE>(g, win[2], 2), m.template out<EDGE>(g, win[3], 3)));
}

// adds (SIGN = 1) or retires (SIGN = -1) a row of the window in the column sums V.  In a dirty row (one the warp
// voted to hold a NaN / inf / huge cell) such cells stay out of V and are counted in C instead.
template <int SIGN>
__device__ __forceinline__ void bs_update(double (&V)[4], unsigned (&C)[4], const float (&v)[4], bool dirty, float thr) {
    if (!dirty) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if constexpr (SIGN > 0) V[j] += (double)v[j]; else V[j] -= (double)v[j];
        }
    } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const bool isnan_ = v[j] != v[j];
            const bool big = !isnan_ && !(fabsf(v[j]) < thr);
            const double d = (isnan_ || big) ? 0.0 : (double)v[j];
            const unsigned c = isnan_ ? 1u : (big ? 0x10000u : 0u);
            if constexpr (SIGN > 0) { V[j] += d; C[j] += c; } else { V[j] -= d; C[j] -= c; }
        }
    }
}

// M: BoxConvolve or BoxNanMean
template <int RX, int NW, template <int> class M>
__global__ void __launch_bounds__((NW + 1) * 32, 2)
box_stream_kernel(const __grid_constant__ CUtensorMap tmap, const float *__restrict__ in, int64_t in_pitch_elems,
                  float *__restrict__ out, int64_t out_pitch_elems, const BoxGeom g) {
    using S = BoxShape<RX, NW>;
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
                for (int e0 = 0; e0 < n_in; e0 += kBoxRows) {
                    mbar_wait(&empty[stage], lap ^ 1u);  // a fresh barrier passes the first lap
                    const bool leaving = e0 + kBoxRows - 1 >= kh - 1;
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
        const bool store_ok = emits && in_raster;                           // out-of-raster lanes never vote a row dirty
        const M<RX> m(g, x, in_raster);
        float *optr = out + y0 * out_pitch_elems + x;

        double V[4] = {0.0, 0.0, 0.0, 0.0};
        unsigned C[4] = {0u, 0u, 0u, 0u};   // lo 16 bits: NaN cells in the column window, hi 16: infinite / huge
        uint32_t dirty = 0;                  // bit i: the row added i rows ago held a NaN / inf / huge cell (this warp)
        const int n_in = (int)(y1 - y0) + kh - 1;
        for (int e0 = 0; e0 < n_in; e0 += kBoxRows) {
            mbar_wait(&full[stage], lap);
            const float *se = ring + (size_t)stage * kStageCells + off;   // entering rows
            const float *sl = se + S::kHalfCells;                          // leaving rows
            bool done = false;
            if (e0 >= kh - 1 && e0 + kBoxRows <= n_in && (dirty & win_mask) == 0u) {
                // ---- fast path: window complete, 4 rows enter, 4 rows are emitted, 4 rows leave; neither
                // the window nor the entering rows hold a NaN / inf / huge cell inside the raster
                float nv[kBoxRows][4];
#pragma unroll
                for (int i = 0; i < kBoxRows; ++i) bs_row<true>(m, se + i * S::kBoxW, nv[i]);
                const float amax = bs_amax3(bs_amax3(bs_amax4(nv[0]), nv[1][0], nv[1][1]),
                                            bs_amax3(bs_amax4(nv[2]), nv[1][2], nv[1][3]), bs_amax4(nv[3]));
                if (!__any_sync(0xffffffffu, in_raster && !(amax < thr))) {
                    float ov[kBoxRows][4];
#pragma unroll
                    for (int i = 0; i < kBoxRows; ++i) bs_row<true>(m, sl + i * S::kBoxW, ov[i]);
                    // column sums of output row i: V_i = V_{i-1} - old_{i-1} + new_i
                    double P[kBoxRows][4];
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        double acc = V[j];
#pragma unroll
                        for (int i = 0; i < kBoxRows; ++i) {
                            const double d = (i == 0) ? (double)nv[0][j] : ((double)nv[i][j] - (double)ov[i > 0 ? i - 1 : 0][j]);
                            acc += d;
                            P[i][j] = acc;
                        }
                        V[j] = acc - (double)ov[kBoxRows - 1][j];
                    }
                    double win[kBoxRows][4];
                    bs_lanesum<RX, kBoxRows, double>(P, win);
#pragma unroll
                    for (int i = 0; i < kBoxRows; ++i) {
                        if (store_ok) {
                            if (!m.edge_warp) bs_store<false>(m, optr, g, win[i]);   // warp-uniform
                            else bs_store<true>(m, optr, g, win[i]);
                        }
                        optr += out_pitch_elems;
                    }
                    dirty <<= kBoxRows;
                    done = true;
                }
            }
            if (!done) {
                // ---- row by row: lead-in rows (nothing to emit yet), the last rows of a task, and windows
                // or entering rows with NaN / inf / huge cells (kept out of V, counted in C)
                for (int i = 0; i < kBoxRows; ++i) {
                    const int e = e0 + i;
                    if (e >= n_in) break;
                    float v[4];
                    bs_row<false>(m, se + i * S::kBoxW, v);
                    const bool row_dirty = __any_sync(0xffffffffu, in_raster && !(bs_amax4(v) < thr));
                    dirty = (dirty << 1) | (row_dirty ? 1u : 0u);
                    bs_update<1>(V, C, v, row_dirty, thr);
                    if (e < kh - 1) continue;   // window not complete yet

                    // emit output row y = y0 + e - (kh - 1)
                    const bool win_dirty = (dirty & bs_bits(kh)) != 0u;
                    double P1[1][4] = {{V[0], V[1], V[2], V[3]}}, w1[1][4];
                    bs_lanesum<RX, 1, double>(P1, w1);
                    float res[4];
#pragma unroll
                    for (int j = 0; j < 4; ++j)
                        res[j] = m.edge_warp ? m.template out<true>(g, w1[0][j], j) : m.template out<false>(g, w1[0][j], j);
                    if (win_dirty) {   // warp-uniform
                        unsigned C1[1][4] = {{C[0], C[1], C[2], C[3]}}, wc[1][4];
                        bs_lanesum<RX, 1, unsigned>(C1, wc);
                        const int64_t y = y0 + e - (kh - 1);
#pragma unroll
                        for (int j = 0; j < 4; ++j)
                            m.finish_exceptional(res[j], j, w1[0][j], wc[0][j], store_ok, in, in_pitch_elems, g, y, x);
                    }
                    if (store_ok) __stcs(reinterpret_cast<float4 *>(optr), make_float4(res[0], res[1], res[2], res[3]));
                    optr += out_pitch_elems;

                    // retire input row e - (kh - 1), the oldest row of the window
                    float vo[4];
                    bs_row<false>(m, sl + i * S::kBoxW, vo);
                    bs_update<-1>(V, C, vo, (dirty >> (kh - 1)) & 1u, thr);
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[stage]);
            if (++stage == g.stages) { stage = 0; lap ^= 1u; }
        }
    }
}

template <int RX, template <int> class M>
static int launch_box_stream(const CUtensorMap &tmap, const float *in, int64_t in_pitch, float *out, int64_t out_pitch,
                             int64_t H, int64_t W, int kh, double w, cudaStream_t s) {
    using S = BoxShape<RX, kBsWarps>;
    BoxGeom g;
    g.H = H; g.W = W; g.kh = kh; g.ry = kh / 2; g.w = w;
    g.n_cells = (double)(kh * (2 * RX + 1));
    g.n_tiles = (int)((W + S::kTileOutW - 1) / S::kTileOutW);
    // 3 stages up to radius 2 and 4 above, at most 2 CTAs per SM, row segments for 4 waves of tasks: the fastest
    // setting of a sweep of 2 .. 6 stages, 1 / 2 CTAs per SM and 2 .. 8 waves at k = 5, 9, 15, 25 over a 32768^2
    // DEM, run on a B200 when the kernel was written and not repeated on the H100
    g.stages = RX <= 2 ? 3 : 4;
    const size_t smem = (size_t)g.stages * (2 * S::kHalfBytes + 2 * sizeof(uint64_t));
    static_assert(4 * (2 * S::kHalfBytes + 2 * sizeof(uint64_t)) <= (kSmemPerSm - 2 * kSmemReservedPerCta) / 2 - 256,
                  "4 stages for each of 2 CTAs per SM");
    auto kern = box_stream_kernel<RX, kBsWarps, M>;
    int64_t resident;
    if (const int rc = resident_ctas(kern, (kBsWarps + 1) * 32, smem, 2, &resident)) return rc;
    // segments: tall enough that the kh - 1 lead-in rows stay a small overhead, (rows + kh - 1) a
    // multiple of 4 so that only the raster's last segment ends in a partial batch
    const int64_t seg_rows = pick_seg_rows(H, g.n_tiles, resident, 12 * (int64_t)kh, kh - 1, kBoxRows, 4);
    g.seg_rows = (int)seg_rows;
    g.n_segs = (int)((H + seg_rows - 1) / seg_rows);
    const int64_t n_tasks = (int64_t)g.n_tiles * g.n_segs;
    return launch(kern, resident < n_tasks ? resident : n_tasks, (kBsWarps + 1) * 32, smem, s, kRunningBox, tmap, in,
                  in_pitch / 4, out, out_pitch / 4, g);
}

// Calls f(std::integral_constant<int, R>{}) with R = rx for rx in 1 .. 12 (the first R tried is R0); false for any
// other rx.
template <int R0 = 1, typename F> static bool with_radius(int rx, F &&f) {
    if constexpr (R0 > kBsMaxK / 2) return false;
    else return rx == R0 ? f(std::integral_constant<int, R0>{}) : with_radius<R0 + 1>(rx, f);
}

bool try_running_box(BoxMode mode, double w, const float *in, int64_t in_pitch, float *out, int64_t out_pitch,
                     int64_t H, int64_t W, int kh, int kw, cudaStream_t s, int *rc) {
    if (kh > kBsMaxK || kw > kBsMaxK || kh < 1 || kw < 3 || (kw & 1) == 0 || (kh & 1) == 0) return false;
    if (W % 4 != 0 || out_pitch % 16 != 0 || (reinterpret_cast<uintptr_t>(out) & 15)) return false;
    if (H >= (1LL << 31) - 64 || W >= (1LL << 31) - 4096) return false;
    return with_radius(kw / 2, [&](auto R) {
        CUtensorMap tmap;
        if (!make_tensor_map_2d(&tmap, in, in_pitch, H, W, XRS_F32, BoxShape<R, kBsWarps>::kBoxW, kBoxRows))
            return false;   // TMA cannot describe the raster: the tiled kernels take it
        *rc = mode == BoxMode::kConvolve
                  ? launch_box_stream<R, BoxConvolve>(tmap, in, in_pitch, out, out_pitch, H, W, kh, w, s)
                  : launch_box_stream<R, BoxNanMean>(tmap, in, in_pitch, out, out_pitch, H, W, kh, w, s);
        return true;
    });
}

}  // namespace xrs

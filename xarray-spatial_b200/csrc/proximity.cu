// proximity.cu -- proximity / allocation / direction (proximity.py:401-647) as an exact nearest-target
// transform: a row pass picks each cell's nearest target within its own row, a column pass picks the nearest
// of the rows' picks (proximity_envelope.cuh), and the epilogue writes the mode's output.  Everything that
// selects a target is float64; the output values follow the reference's own roundings (DESIGN.md section 4.7).
#include <math.h>

#include "common.cuh"
#include "proximity_envelope.cuh"

namespace xrs {
namespace {

using namespace prox;

constexpr int kRowThreads = 256;
constexpr double kDegToRad = 3.141592653589793 / 180.0;   // np.radians
constexpr int kNoTarget = 0x7fffffff;

struct TargetRule {
    const double *values;   // sorted, NaN-free; nullptr: nonzero and finite cells are targets
    int n;
};

template <typename T> __device__ __forceinline__ bool is_target(T raw, const TargetRule &rule) {
    const double v = (double)raw;   // how NumPy compares the cell with float64 target values
    if (rule.values == nullptr) return v != 0.0 && isfinite(v);
    int a = 0, z = rule.n;
    while (a < z) {
        const int m = (a + z) >> 1;
        if (rule.values[m] < v) a = m + 1; else z = m;
    }
    return a < rule.n && rule.values[a] == v;
}

// The row pass key of target column t for cell column c: smaller is nearer.
template <int M> __device__ __forceinline__ double row_key(const double *X, const double *lam, int t, int c) {
    if (M == kGreatCircle) return -cos(lam[t] - lam[c]);   // the haversine grows with 1 - cos(dlon)
    const double dx = X[t] - X[c];
    return M == kEuclidean ? dx * dx : fabs(dx);
}

// One CTA per row.  Right-to-left: the first target at or after each column (inclusive min-scan), written to
// ridx.  Left-to-right: the last target at or before it (max-scan); the nearer of the two, the left one on a
// tie; a target cell keeps itself.  The great circle also weighs the row's first and last target, the candidates
// across the antimeridian.
template <typename T, int M>
__global__ void __launch_bounds__(kRowThreads) prox_row_kernel(const void *in, int64_t in_pitch, int64_t W,
                                                               TargetRule rule, const double *X, const double *lam,
                                                               int32_t *ridx) {
    __shared__ int s_warp[kRowThreads / 32];
    __shared__ int s_carry, s_lcarry, s_last;   // the two scans' carries, the row's last target
    const int64_t r = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int32_t *row = ridx + r * W;
    const int ntiles = (int)((W + kRowThreads - 1) / kRowThreads);
    if (tid == 0) { s_carry = kNoTarget; s_lcarry = -1; s_last = -1; }
    __syncthreads();
    for (int k = ntiles - 1; k >= 0; --k) {
        const int c = k * kRowThreads + tid;
        const bool tg = c < W && is_target(Cells<T>{(const char *)in, in_pitch}(r, c), rule);
        int v = tg ? c : kNoTarget;
        if (M == kGreatCircle) {
            const int mx = __reduce_max_sync(0xffffffffu, tg ? c : -1);
            if (lane == 0 && mx >= 0) atomicMax(&s_last, mx);
        }
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_down_sync(0xffffffffu, v, o);
            if (lane + o < 32) v = min(v, y);
        }
        if (lane == 0) s_warp[warp] = v;
        __syncthreads();
        for (int w = warp + 1; w < kRowThreads / 32; ++w) v = min(v, s_warp[w]);
        v = min(v, s_carry);
        if (c < W) row[c] = v;
        __syncthreads();
        if (tid == 0) s_carry = v;   // thread 0 holds the whole tile's minimum
        __syncthreads();
    }
    const int first = s_carry, last = s_last;
    for (int k = 0; k < ntiles; ++k) {
        const int c = k * kRowThreads + tid;
        const int right = c < W ? row[c] : kNoTarget;
        int v = right == c ? c : -1;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, v, o);
            if (lane >= o) v = max(v, y);
        }
        if (lane == 31) s_warp[warp] = v;
        __syncthreads();
        for (int w = 0; w < warp; ++w) v = max(v, s_warp[w]);
        v = max(v, s_lcarry);
        if (c < W && right == c) {
            row[c] = c;   // a target is its own nearest target, also when a wrap-around one ties it
        } else if (c < W) {
            // candidates in increasing column order; a later one replaces only a strictly farther one
            const int cand[4] = {M == kGreatCircle ? first : kNoTarget, v, right, M == kGreatCircle ? last : -1};
            int best = -1;
            double bk = 0.0;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int t = cand[q];
                if (t < 0 || t >= W) continue;
                const double key = row_key<M>(X, lam, t, c);
                if (best < 0 || key < bk) { best = t; bk = key; }
            }
            row[c] = best;
        }
        __syncthreads();
        if (tid == kRowThreads - 1) s_lcarry = v;
        __syncthreads();
    }
}

// Per-row / per-column tables: the great circle's cos / sin of each latitude and each longitude in radians.
__global__ void prox_tables_kernel(const double *X, const double *Y, int64_t H, int64_t W, double *cosl,
                                   double *sinl, double *lam) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < H + W; k += (int64_t)gridDim.x * blockDim.x) {
        if (k < H) {
            const double p = Y[k] * kDegToRad;
            cosl[k] = cos(p);
            sinl[k] = sin(p);
        } else {
            lam[k - H] = X[k - H] * kDegToRad;
        }
    }
}

struct ProxArgs {
    const void *in;
    int64_t in_pitch, H, W, out_pitch;
    float *out;
    const double *X, *Y;
    double max_distance;
    int mode;
};

template <int M> __device__ __forceinline__ Column<M> column_of(const Column<M> &proto, int64_t c) {
    Column<M> col = proto;
    col.c = c;
    return col;
}

template <int M> __global__ void prox_build_kernel(Column<M> proto) {
    const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= proto.W) return;
    build_band(column_of(proto, c), (int)blockIdx.y);
}

template <int M> __global__ void prox_merge_kernel(Column<M> proto) {
    const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= proto.W) return;
    merge_bands(column_of(proto, c));
}

// great_circle_distance (proximity.py:135-219) with the target as the first point
__device__ __forceinline__ double haversine(double x1, double x2, double y1, double y2) {
    const double lat1 = y1 * kDegToRad, lon1 = x1 * kDegToRad, lat2 = y2 * kDegToRad, lon2 = x2 * kDegToRad;
    const double dlon = lon2 - lon1, dlat = lat2 - lat1;
    const double s1 = sin(dlat / 2.0), s2 = sin(dlon / 2.0);
    const double a = s1 * s1 + cos(lat1) * cos(lat2) * (s2 * s2);
    return 6378137.0 * 2.0 * asin(sqrt(a));
}

// _calc_direction (proximity.py:238-258) from the cell (x1, y1) to the target (x2, y2)
__device__ __forceinline__ float direction_deg(double x1, double x2, double y1, double y2) {
    if (x1 == x2 && y1 == y2) return 0.0f;
    const double x = x2 - x1, y = y2 - y1;
    double d = atan2(-y, x) * 57.29578;
    if (d < 0.0) d = 90.0 - d;
    else if (d > 90.0) d = 360.0 - d + 90.0;
    else d = 90.0 - d;
    return (float)d;
}

template <typename T, int M> __global__ void prox_query_kernel(Column<M> proto, ProxArgs a) {
    const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= proto.W) return;
    const Column<M> col = column_of(proto, c);
    const double md2 = a.max_distance * a.max_distance;
    query_band(col, (int)blockIdx.y, [&](int64_t i, int64_t r) {
        float res = __int_as_float(0x7fc00000);
        const bool self = col.target(i) == (int32_t)c;   // a target is its own nearest target
        if (self) r = i;
        if (r >= 0) {
            const int64_t t = self ? c : col.target(r);
            const double xt = a.X[t], yt = a.Y[r], xc = a.X[c], yc = a.Y[i];
            double d;
            if (M == kEuclidean) {
                const double dx = xt - xc, dy = yt - yc;
                d = sqrt(dx * dx + dy * dy);
            } else if (M == kManhattan) {
                d = fabs(xt - xc) + fabs(yt - yc);
            } else {
                d = haversine(xt, xc, yt, yc);
            }
            const float f = (float)d;
            const float sq = f * f;   // the reference keeps the squared float32 distance
            if (self || md2 >= (double)sq) {
                if (a.mode == XRS_PROX_DISTANCE) res = self ? 0.0f : (float)sqrt((double)sq);
                else if (a.mode == XRS_PROX_ALLOCATION) res = (float)Cells<T>{(const char *)a.in, a.in_pitch}(r, t);
                else res = self ? 0.0f : direction_deg(xc, xt, yc, yt);
            }
        }
        a.out[i * a.out_pitch + c] = res;
    });
}

// Scratch layout: ridx and stk (H x W int32 each), the band arrays (3 nb + 1 rows of W int32), the great-circle
// tables (2 H + W doubles), each 256-byte aligned.
struct Layout {
    int64_t band_rows, nb, ridx, stk, blo, bhi, bprev, boff, cosl, sinl, lam, total;
};

Layout layout(int64_t H, int64_t W, int64_t band_rows) {
    Layout L;
    if (band_rows <= 0) {   // about a million (band, column) threads for the band phases, bands of >= 32 rows
        const int64_t want_bands = (((int64_t)1 << 20) + W - 1) / W;
        band_rows = (H + want_bands - 1) / want_bands;
        if (band_rows < 32) band_rows = 32;
    }
    if (band_rows > H) band_rows = H;
    if ((H + band_rows - 1) / band_rows > 65535) band_rows = (H + 65534) / 65535;   // bands are a grid dimension
    L.band_rows = band_rows;
    L.nb = (H + band_rows - 1) / band_rows;
    const int64_t cells = align256(H * W * 4), band = align256(L.nb * W * 4);
    L.ridx = 0;
    L.stk = L.ridx + cells;
    L.blo = L.stk + cells;
    L.bhi = L.blo + band;
    L.bprev = L.bhi + band;
    L.boff = L.bprev + band;
    L.cosl = L.boff + align256((L.nb + 1) * W * 4);
    L.sinl = L.cosl + align256(H * 8);
    L.lam = L.sinl + align256(H * 8);
    L.total = L.lam + align256(W * 8);
    return L;
}

int check_shape(int64_t H, int64_t W, int band_rows) {
    XRS_REQUIRE(H >= 0 && W >= 0, "negative raster shape");
    XRS_REQUIRE(H < INT32_MAX && W < INT32_MAX, "rows and columns must each be below 2^31");
    XRS_REQUIRE(band_rows >= 0, "band_rows must be >= 0 (0: the library's choice)");
    if (H > 0 && W > 0 && H > (INT64_MAX / 16) / W) {
        set_error("a %lld x %lld raster's scratch does not fit in 64-bit sizes", (long long)H, (long long)W);
        return XRS_ENOMEM;
    }
    return XRS_OK;
}

template <typename T, int M> int run(const void *in, int64_t in_pitch, int64_t H, int64_t W, const double *x,
                                     const double *y, TargetRule rule, double max_distance, int mode, float *out,
                                     int64_t out_pitch, char *scratch, const Layout &L,
                                     cudaStream_t s) {
    int32_t *ridx = (int32_t *)(scratch + L.ridx);
    double *cosl = (double *)(scratch + L.cosl), *sinl = (double *)(scratch + L.sinl),
           *lam = (double *)(scratch + L.lam);
    if (M == kGreatCircle) {
        int64_t g = (H + W + 255) / 256;
        if (g > 4096) g = 4096;
        prox_tables_kernel<<<(unsigned)g, 256, 0, s>>>(x, y, H, W, cosl, sinl, lam);
        XRS_CUDA(cudaGetLastError());
    }
    int rc = launch(prox_row_kernel<T, M>, H, kRowThreads, 0, s, kProximity, in, in_pitch, W, rule, x,
                    (const double *)lam, ridx);
    if (rc) return rc;
    Column<M> col;
    col.ridx = ridx;
    col.stk = (int32_t *)(scratch + L.stk);
    col.blo = (int32_t *)(scratch + L.blo);
    col.bhi = (int32_t *)(scratch + L.bhi);
    col.bprev = (int32_t *)(scratch + L.bprev);
    col.boff = (int32_t *)(scratch + L.boff);
    col.X = x;
    col.Y = y;
    col.cosl = cosl;
    col.sinl = sinl;
    col.lam = lam;
    col.H = H;
    col.W = W;
    col.c = 0;
    col.band_rows = L.band_rows;
    col.nb = (int)L.nb;
    const unsigned gx = (unsigned)((W + 127) / 128);
    prox_build_kernel<M><<<dim3(gx, (unsigned)L.nb), 128, 0, s>>>(col);
    XRS_CUDA(cudaGetLastError());
    prox_merge_kernel<M><<<(unsigned)((W + 63) / 64), 64, 0, s>>>(col);
    XRS_CUDA(cudaGetLastError());
    ProxArgs a{in, in_pitch, H, W, out_pitch / 4, out, x, y, max_distance, mode};
    prox_query_kernel<T, M><<<dim3(gx, (unsigned)L.nb), 128, 0, s>>>(col, a);
    XRS_CUDA(cudaGetLastError());
    return XRS_OK;
}

template <typename T> int run_metric(int metric, const void *in, int64_t in_pitch, int64_t H, int64_t W,
                                     const double *x, const double *y, TargetRule rule, double max_distance,
                                     int mode, float *out, int64_t out_pitch, char *scratch, const Layout &L,
                                     cudaStream_t s) {
    if (metric == kGreatCircle)
        return run<T, kGreatCircle>(in, in_pitch, H, W, x, y, rule, max_distance, mode, out, out_pitch, scratch, L, s);
    if (metric == kManhattan)
        return run<T, kManhattan>(in, in_pitch, H, W, x, y, rule, max_distance, mode, out, out_pitch, scratch, L, s);
    return run<T, kEuclidean>(in, in_pitch, H, W, x, y, rule, max_distance, mode, out, out_pitch, scratch, L, s);
}

}  // namespace
}  // namespace xrs

using namespace xrs;

extern "C" int xrs_proximity_scratch_bytes(int64_t H, int64_t W, int band_rows, int64_t *bytes) {
    XRS_REQUIRE(bytes != nullptr, "NULL pointer");
    const int rc = check_shape(H, W, band_rows);
    if (rc) return rc;
    *bytes = (H > 0 && W > 0) ? layout(H, W, band_rows).total : 0;
    return XRS_OK;
}

extern "C" int xrs_proximity(const void *in, int in_dtype, int64_t in_pitch, int64_t H, int64_t W, const double *x,
                             const double *y, const double *targets, int n_targets,
                             double max_distance, int metric, int mode, float *out, int64_t out_pitch,
                             void *scratch, int64_t scratch_bytes, int band_rows, xrs_stream_t s) {
    int rc = check_shape(H, W, band_rows);
    if (rc) return rc;
    XRS_REQUIRE(metric == XRS_METRIC_EUCLIDEAN || metric == XRS_METRIC_GREAT_CIRCLE || metric == XRS_METRIC_MANHATTAN,
                "unknown distance metric");
    XRS_REQUIRE(mode == XRS_PROX_DISTANCE || mode == XRS_PROX_ALLOCATION || mode == XRS_PROX_DIRECTION,
                "unknown proximity mode");
    XRS_REQUIRE(n_targets >= 0 && (n_targets == 0 || targets != nullptr), "bad target list");
    if (H == 0 || W == 0) return XRS_OK;
    XRS_REQUIRE(in && out && x && y, "NULL pointer");
    XRS_TRY(check_cells_arg(in, in_dtype, kRasterCells, in_pitch, W));
    XRS_TRY(check_out_pitch(out_pitch, 4, W));
    const Layout L = layout(H, W, band_rows);
    XRS_TRY(check_scratch(scratch, scratch_bytes, L.total, "xrs_proximity_scratch_bytes"));
    const TargetRule rule{targets, n_targets};
    return with_cell_type(kRasterCells, in_dtype, [&](auto z) {
        return run_metric<decltype(z)>(metric, in, in_pitch, H, W, x, y, rule, max_distance, mode, out, out_pitch,
                                       (char *)scratch, L, (cudaStream_t)s);
    });
}

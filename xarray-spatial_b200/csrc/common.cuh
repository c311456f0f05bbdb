// common.cuh -- shared host/device helpers for libxrs_b200 (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <limits.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <type_traits>

#include "../../include/xrs_b200.h"

namespace xrs {

// ----------------------------------------------------------------------------- errors
void set_error(const char *fmt, ...);
int cuda_fail(cudaError_t e, const char *what);

// Which kernel a launch ran (xrs_debug_last_used_tma reports it; the codes are listed in xrs_b200.h).
enum LaunchKind : int {
    kStripCpAsync = 0,  // 3x3 strip kernel, per-warp cp.async ring
    kStripTma = 1,      // 3x3 strip kernel, CTA-wide TMA ring
    kIngestTma = 2,     // 3x3 TMA strip kernel reading int16 / uint16 / int32 / float64 cells
    kRunningBox = 3,    // running-box convolve_2d / focal.apply mean
    kConvTiled = 4,     // tiled k x k convolve
    kConvDirect = 5,    // bounds-checked convolve
    kFocalFused = 6,    // every requested focal statistic in one pass
    kFocalTiled = 7,    // tiled single focal statistic
    kFocalDirect = 8,   // bounds-checked single focal statistic
    kZonalHash = 9,     // zonal group-by
    kZonalPair = 10,    // zonal (zone, value) pair count
    kConvWide = 11,     // convolve over a window beyond the tiled kernels (conv.cu, "wide windows")
    kFocalWide = 12,    // single focal statistic over such a window
    kFocalWideFused = 13,  // every requested focal statistic over such a window
    kProximity = 14,    // proximity / allocation / direction row pass (proximity.cu)
    kClassify = 15,     // classify per-cell bin / membership pass (classify.cu)
};

struct LaunchInfo {  // for tests / profiling: what the last launch on this thread chose
    int kind;        // a LaunchKind
    int grid, block, smem_bytes;
};
LaunchInfo &last_launch_info();

#define XRS_CUDA(call)                                              \
    do {                                                            \
        cudaError_t _e = (call);                                    \
        if (_e != cudaSuccess) return ::xrs::cuda_fail(_e, #call);  \
    } while (0)

#define XRS_REQUIRE(cond, msg)                     \
    do {                                           \
        if (!(cond)) {                             \
            ::xrs::set_error("%s", msg);           \
            return XRS_EINVAL;                     \
        }                                          \
    } while (0)

// returns the status of a call that failed
#define XRS_TRY(call)                  \
    do {                               \
        const int _rc = (call);        \
        if (_rc != XRS_OK) return _rc; \
    } while (0)

// XRS_EINVAL with a message unless kh and kw are odd and 1 .. 2047: the windows of convolve and the focal
// statistics (conv.cu)
int check_window(int kh, int kw);

// Slope, aspect, curvature or hillshade (op 0-3, an xrs_op) on a device raster of in_dtype cells: float32, or
// int16 / uint16 / int32 / float64 converted in registers; float32 out (surface.cu).  p: slope {csx, csy};
// curvature {cellsize}; hillshade {azimuth, altitude}; aspect takes none.
int surface_op(int op, const void *in, int in_dtype, int64_t in_pitch, float *out, int64_t out_pitch, int64_t H,
               int64_t W, const double *p, cudaStream_t s);

// The running box (box_stream.cu), O(1) work per cell for any window: convolve_2d with every tap the weight w, or
// focal.apply's mean over an all-ones window (w = 1 / (kh kw)).  Returns false without launching when it cannot
// take the window (odd sides, kh <= 25, 3 <= kw <= 25) or the raster; otherwise *rc is the launch's status.
enum class BoxMode { kConvolve, kNanMean };
bool try_running_box(BoxMode mode, double w, const float *in, int64_t in_pitch, float *out, int64_t out_pitch,
                     int64_t H, int64_t W, int kh, int kw, cudaStream_t s, int *rc);

// cached per-device properties
int sm_count(int device = -1);

// Shared memory of an H100 SM: 228 KB, at most 227 KB of it for one CTA, 1 KB reserved per resident CTA.
constexpr size_t kSmemPerSm = 228 * 1024, kSmemPerCtaMax = 227 * 1024, kSmemReservedPerCta = 1024;

// Persistent kernels: sets `kernel`'s dynamic shared-memory limit to `smem`, then *resident = the CTAs of
// `threads` threads that fit on the device at once, between 1 and max_per_sm per SM.
int resident_ctas(const void *kernel, int threads, size_t smem, int max_per_sm, int64_t *resident);
template <typename... P>
int resident_ctas(void (*kernel)(P...), int threads, size_t smem, int max_per_sm, int64_t *resident) {
    return resident_ctas(reinterpret_cast<const void *>(kernel), threads, smem, max_per_sm, resident);
}

// Records the launch in last_launch_info(), launches `kernel` and reports a launch error.
template <typename... P, typename... A>
int launch(void (*kernel)(P...), int64_t grid, int threads, size_t smem, cudaStream_t stream, LaunchKind kind,
           const A &...args) {
    last_launch_info() = {kind, (int)grid, threads, (int)smem};
    kernel<<<(unsigned)grid, threads, smem, stream>>>(args...);
    XRS_CUDA(cudaGetLastError());
    return XRS_OK;
}

// Encodes a 2-D tiled tensor map over a row-major (H, W) raster of `dtype` cells (float32, float64, int32,
// int16 or uint16).  Float cells beyond the raster read as NaN (the raster-edge semantics of the reference's
// `boundary=np.nan` overlap, slope.py:94-97); integer cells read as 0, and their kernels substitute NaN from
// the cell coordinates.  Returns false if TMA cannot describe the raster (base / pitch not 16-byte aligned,
// ...); callers then use kernels that load without TMA.
bool make_tensor_map_2d(CUtensorMap *map, const void *base, int64_t pitch_bytes, int64_t H, int64_t W,
                        xrs_dtype dtype, int box_w, int box_h);

// ----------------------------------------------------------------------------- raster arguments
// Bytes per cell of an xrs_dtype code; 0 for an unknown code.
inline int cell_size(int dtype) {
    switch (dtype) {
        case XRS_I8: case XRS_U8: case XRS_BOOL: return 1;
        case XRS_I16: case XRS_U16: return 2;
        case XRS_F32: case XRS_I32: case XRS_U32: return 4;
        case XRS_F64: case XRS_I64: case XRS_U64: return 8;
        default: return 0;
    }
}

// The cell sets of xrs_b200.h: the raster set (F32, F64, I32, I64, I16, U16) and the zonal set (every code).
struct RasterCells { static constexpr bool kAll = false; };
struct ZonalCells { static constexpr bool kAll = true; };
constexpr RasterCells kRasterCells{};
constexpr ZonalCells kZonalCells{};

template <class Set> bool in_cell_set(Set, int dtype) {
    return Set::kAll ? cell_size(dtype) > 0 : (dtype >= XRS_F32 && dtype <= XRS_U16);
}

// Returns f(a value of dtype's C++ type) for a dtype in `set` (XRS_BOOL: bool), else XRS_EINVAL.
template <class Set, class F> int with_cell_type(Set, int dtype, F &&f) {
    switch (dtype) {
        case XRS_F32: return f(float{});
        case XRS_F64: return f(double{});
        case XRS_I32: return f(int32_t{});
        case XRS_I64: return f((long long)0);
        case XRS_I16: return f(int16_t{});
        case XRS_U16: return f(uint16_t{});
    }
    if constexpr (Set::kAll) {
        switch (dtype) {
            case XRS_I8: return f(int8_t{});
            case XRS_U8: return f(uint8_t{});
            case XRS_U32: return f(uint32_t{});
            case XRS_U64: return f((unsigned long long)0);
            case XRS_BOOL: return f(bool{});
        }
    }
    set_error("unknown cell type %d", dtype);
    return XRS_EINVAL;
}

// XRS_EINVAL unless `in` is set, dtype is in `set` and rows of W cells fit in_pitch bytes, a multiple of the cell
// size (typed loads stay aligned).
template <class Set> int check_cells_arg(const void *in, int dtype, Set set, int64_t in_pitch, int64_t W) {
    XRS_REQUIRE(in != nullptr, "NULL input");
    XRS_REQUIRE(in_cell_set(set, dtype), "unknown cell type");
    const int64_t esz = cell_size(dtype);
    XRS_REQUIRE(in_pitch % esz == 0 && in_pitch >= W * esz, "bad input pitch");
    return XRS_OK;
}

// XRS_EINVAL unless rows of W cells of esz bytes fit out_pitch bytes, a multiple of esz.
inline int check_out_pitch(int64_t out_pitch, int64_t esz, int64_t W) {
    XRS_REQUIRE(out_pitch % esz == 0 && out_pitch >= W * esz, "bad output pitch");
    return XRS_OK;
}

// XRS_EINVAL unless `scratch` is set and holds `need` bytes; `query` names the entry point that sizes it.
inline int check_scratch(const void *scratch, int64_t bytes, int64_t need, const char *query) {
    XRS_REQUIRE(scratch != nullptr, "NULL scratch buffer");
    if (bytes < need) {
        set_error("scratch buffer of %lld bytes is too small: this call needs %lld (%s)", (long long)bytes,
                  (long long)need, query);
        return XRS_EINVAL;
    }
    return XRS_OK;
}

// Scratch regions start on 256-byte boundaries.
constexpr int64_t align256(int64_t b) { return (b + 255) & ~(int64_t)255; }

// Grid of a 256-thread grid-stride loop over n items: at most 8 CTAs per SM, at least one.
inline int64_t stride_grid(int64_t n) {
    const int64_t g = (n + 255) / 256, cap = (int64_t)sm_count() * 8;
    return g < 1 ? 1 : (g < cap ? g : cap);
}

// Cell (r, c) of a raster of T cells whose rows are `pitch` bytes apart.
template <typename T> struct Cells {
    const char *base;
    int64_t pitch;
    __device__ T operator()(int64_t r, int64_t c) const { return reinterpret_cast<const T *>(base + r * pitch)[c]; }
};

template <typename T> constexpr xrs_dtype dtype_of() {
    if constexpr (std::is_same_v<T, float>) return XRS_F32;
    else if constexpr (std::is_same_v<T, double>) return XRS_F64;
    else if constexpr (std::is_same_v<T, int>) return XRS_I32;
    else if constexpr (std::is_same_v<T, short>) return XRS_I16;
    else {
        static_assert(std::is_same_v<T, unsigned short>, "no tensor-map element type");
        return XRS_U16;
    }
}

// ----------------------------------------------------------------------------- device PTX
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "XRS_WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra XRS_DONE_%=;\n"
        "bra XRS_WAIT_%=;\n"
        "XRS_DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// TMA: 2-D tiled bulk tensor load global -> shared, completion on an mbarrier.
__device__ __forceinline__ void tma_load_2d(void *dst, const CUtensorMap *map, uint64_t *bar,
                                            int x, int y) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)),
        "l"(map), "r"(smem_u32(bar)), "r"(x), "r"(y)
        : "memory");
}
// same, with an L2 eviction-priority hint (a policy from l2_policy_evict_last)
__device__ __forceinline__ void tma_load_2d_hint(void *dst, const CUtensorMap *map, uint64_t *bar, int x, int y,
                                                 uint64_t policy) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint"
        " [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(smem_u32(dst)),
        "l"(map), "r"(smem_u32(bar)), "r"(x), "r"(y), "l"(policy)
        : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap *map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
// Bulk async store shared -> global (1-D, 16-byte aligned ends, size a multiple of 16), tracked by bulk groups.
__device__ __forceinline__ void bulk_store(void *dst, const void *src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(smem_u32(src)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// every committed bulk group has finished READING shared memory (its global writes may still be in flight)
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// generic-proxy writes to shared memory become visible to the async proxy (bulk copies)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

template <typename T> __device__ __forceinline__ T nan_of();
template <> __device__ __forceinline__ float nan_of<float>() { return __int_as_float(0x7fc00000); }
template <> __device__ __forceinline__ double nan_of<double>() {
    return __longlong_as_double(0x7ff8000000000000LL);
}

__device__ __forceinline__ float rsqrt_approx(float x) {
    float r;
    asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ float rcp_approx(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

// atan(a)/a on a in [0,1] as a degree-7 polynomial in z = a*a (minimax, rel err 1e-7;
// 2.5e-7 evaluated in f32).  The reference evaluates np.arctan in f64 and rounds to f32;
// the parity bar is 1e-5 relative.  SCALE folds a unit conversion into the coefficients.
template <int DEG> __device__ __forceinline__ float atan_poly01(float z) {
    constexpr float k = DEG ? 57.29578f : 1.0f;  // slope.py:75 uses the literal 57.29578
    float p = -4.693183854e-03f * k;
    p = fmaf(p, z, 2.425208207e-02f * k);
    p = fmaf(p, z, -5.948595430e-02f * k);
    p = fmaf(p, z, 9.914263125e-02f * k);
    p = fmaf(p, z, -1.401947061e-01f * k);
    p = fmaf(p, z, 1.996972220e-01f * k);
    p = fmaf(p, z, -3.333199064e-01f * k);
    p = fmaf(p, z, 9.999999010e-01f * k);
    return p;
}

// degrees(atan(sqrt(p))) for p >= 0 (NaN propagates).  One MUFU.RSQ per cell,
// no division: for p > 1 uses atan(s) = pi/2 - atan(1/s) with 1/s = rsqrt(p), folded into the last
// FMA as  a * poly(a^2) + off  with (a, off) = (s, 0) or (-1/s, 90 deg).  p below 1e-30 (slope below
// 6e-14 degrees) evaluates as p * 1e15, far under any tolerance.
__device__ __forceinline__ void atan_sqrt_sel(float p, float &a, float &off) {
    const float r = rsqrt_approx(fmaxf(p, 1e-30f));
    const bool big = p > 1.0f;          // false for NaN -> a = p * r = NaN propagates
    a = big ? -r : p * r;               // +-atan argument in [0, 1]
    off = big ? (1.57079632679489662f * 57.29578f) : 0.0f;
}
__device__ __forceinline__ float atan_sqrt_deg(float p) {
    float a, off;
    atan_sqrt_sel(p, a, off);
    return fmaf(a, atan_poly01<1>(a * a), off);
}

// Compass aspect from the Horn sums X = 8 dz_dx, Y = 8 dz_dy (aspect.py:74-88):
// the reference's (90 - atan2(Y, -X) deg) folded to [0, 360) is atan2(u, v) with u = -X, v = Y,
// folded to [0, 360).  One octant reduction (ratio t of the smaller to the larger magnitude,
// one MUFU.RCP, degree-7 polynomial already scaled to degrees), then compass = K + sigma*atan(t)
// with (K, sigma) picked per octant; sigma is applied to t's sign bit (the polynomial is even in t),
// so the tail is one FMA:  ts * poly(ts^2) + K.  Evaluating the compass angle directly keeps full
// relative accuracy near 0 degrees, where `90 - theta` would cancel.  Flat cells (both sums zero)
// give -1; NaN propagates (selects, not fmin/fmax, pick the operands; the flat test is NaN-safe:
// a NaN sum next to a zero sum is NaN, like atan2(0, NaN) in the reference).  The reciprocal is
// rcp.approx.ftz: it needs normal max(|u|, |v|) <= 2^125 (its result is then a normal float); the
// 3x3 aspect scales larger pairs first (surface_ops.cuh, compass_uv4).
struct CompassPre {
    float ts, K;
    bool flat;
};
// NaN-propagating max / min (FMNMX.NAN): a NaN operand gives NaN, unlike fmaxf / fminf
__device__ __forceinline__ float max_nan(float a, float b) {
    float r;
    asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}
__device__ __forceinline__ float min_nan(float a, float b) {
    float r;
    asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}
__device__ __forceinline__ CompassPre compass_pre(float u, float v) {
    const float au = fabsf(u), av = fabsf(v);
    const bool swap = au > av;                // closer to the +-u axis (east / west)
    const float mx = max_nan(au, av), mn = min_nan(au, av);   // a NaN sum makes both NaN
    const float t = mn * rcp_approx(mx);
    // sigma = sign(u) * sign(v), negated in the swapped octants: flip t's sign bit
    const unsigned sgn = ((__float_as_uint(u) ^ __float_as_uint(v)) & 0x80000000u) ^ (swap ? 0x80000000u : 0u);
    CompassPre c;
    c.ts = __uint_as_float(__float_as_uint(t) ^ sgn);
    const float k_ns = (v > 0.0f) ? ((u < 0.0f) ? 360.0f : 0.0f) : 180.0f;
    const float k_ew = (u > 0.0f) ? 90.0f : 270.0f;
    c.K = swap ? k_ew : k_ns;
    c.flat = mx == 0.0f;                       // false for NaN: atan2(0, NaN) is NaN in the reference, not "flat"
    return c;
}
__device__ __forceinline__ float compass_deg(float u, float v) {
    const CompassPre c = compass_pre(u, v);
    const float r = fmaf(c.ts, atan_poly01<1>(c.ts * c.ts), c.K);
    return c.flat ? -1.0f : r;
}
}  // namespace xrs

// surface.cu -- C-ABI entry points of the 3x3 family (slope, aspect, curvature, hillshade,
// fused suite, focal.mean).  Argument checking and launch geometry live in stencil3.cuh.
#include "surface_ops.cuh"

using namespace xrs;

// Pipeline geometry per operator: ROWS rows per TMA stage, STAGES stages, WARPS consumer warps per CTA,
// CTAs per SM (launch_stencil3), swept with scripts/tune/tune5.cu (output in tune5-h100.txt).  With the
// bulk-store epilogue every single-output float32 operator is fastest, or within 0.3 % of it, at one
// 16-warp CTA per SM with a 4 x 3 ring (100 KB of input in flight plus 64 KB of output staging); the
// float64-output focal means prefer 2 x 4.  On an H100 80GB HBM3 (700 W limit), 32768^2, with the loads'
// evict_last hint, these kernels move 0.84-0.85 of the 3.35 TB/s data sheet, 0.93-0.94 of the card's
// measured cudaMemcpy rate (3039-3046 GB/s); focal.mean f64 moves 0.88 / 0.97.  The 4-output suite keeps the
// register-store epilogue (its staging does not fit next to an 8 x 2 ring, and the smaller geometries where
// it fits were not faster with it).
#define XRS_CFG_LIGHT 4, 3, 16, 1     /* hillshade, curvature, focal.mean */
#define XRS_CFG_CONV3 4, 3, 16, 1     /* 3x3 convolution */
#define XRS_CFG_SLOPE_SQ 4, 3, 16, 1  /* slope, square cells */
#define XRS_CFG_SLOPE 4, 3, 16, 1     /* slope, csx != csy */
#define XRS_CFG_ASPECT 4, 3, 16, 1    /* aspect: the most arithmetic per cell */
#define XRS_CFG_SUITE 8, 2, 12, 1     /* ~145 registers per thread: one 12-warp CTA per SM, register stores */
#define XRS_CFG_F64 2, 4, 16, 1       /* 8-byte cells: focal.mean f64 */
#define XRS_CFG_F32_F64 2, 4, 16, 1   /* float32 in, float64 out (12 B/cell) */

// 3x3 kernels of convolve_2d take the warp-strip path (called from conv.cu)
int xrs_conv3_strip(const float *in, int64_t in_pitch, float *out, int64_t out_pitch, int64_t H, int64_t W,
                    const double *kernel, cudaStream_t s) {
    Conv3Op::Params p;
    for (int i = 0; i < 9; ++i) p.w[i] = kernel[i];
    float *outs[1] = {out};
    return launch_stencil3<Conv3Op, XRS_CFG_CONV3>(in, in_pitch, p, outs, out_pitch, H, W, s);
}

template <typename T, typename TOUT, int ROWS, int STAGES, int WARPS, int CTAS>
static int focal_mean_impl(const T *in, int64_t in_pitch, TOUT *out, int64_t out_pitch, int64_t H, int64_t W,
                           const double *excludes, int n_ex, xrs_stream_t s) {
    using Op = FocalMeanOp<T, TOUT, false>;
    using OpEx = FocalMeanOp<T, TOUT, true>;
    static_assert(sizeof(typename Op::Params) == sizeof(typename OpEx::Params), "same parameter block");
    XRS_REQUIRE(n_ex >= 0 && n_ex <= Op::kMaxEx, "at most 8 exclude values are supported");
    XRS_REQUIRE(n_ex == 0 || excludes != nullptr, "excludes is NULL");
    typename OpEx::Params p;
    p.n_ex = 0;
    p.ex_nan = 0;
    for (int i = 0; i < Op::kMaxEx; ++i) p.ex[i] = 0.0;
    for (int i = 0; i < n_ex; ++i) {
        if (excludes[i] != excludes[i]) p.ex_nan = 1;
        else p.ex[p.n_ex++] = excludes[i];
    }
    TOUT *outs[1] = {out};
    if (p.n_ex > 0 || !p.ex_nan) return launch_stencil3<OpEx, ROWS, STAGES, WARPS, CTAS>(in, in_pitch, p, outs, out_pitch, H, W, (cudaStream_t)s);
    typename Op::Params q;
    memcpy(&q, &p, sizeof(q));
    return launch_stencil3<Op, ROWS, STAGES, WARPS, CTAS>(in, in_pitch, q, outs, out_pitch, H, W, (cudaStream_t)s);
}

extern "C" {

int xrs_slope_f32(const float *in, int64_t in_pitch, float *out, int64_t out_pitch, int64_t H, int64_t W,
                  double cellsize_x, double cellsize_y, xrs_stream_t s) {
    const SlopeOp::Params p = SlopeParams::make(cellsize_x, cellsize_y);
    float *outs[1] = {out};
    if (p.rxy == 1.0)  // square cells: same arithmetic minus the multiplication by 1
        return launch_stencil3<SlopeSqOp, XRS_CFG_SLOPE_SQ>(in, in_pitch, p, outs, out_pitch, H, W, (cudaStream_t)s);
    return launch_stencil3<SlopeOp, XRS_CFG_SLOPE>(in, in_pitch, p, outs, out_pitch, H, W,
                                                          (cudaStream_t)s);
}

int xrs_aspect_f32(const float *in, int64_t in_pitch, float *out, int64_t out_pitch, int64_t H, int64_t W,
                   xrs_stream_t s) {
    AspectOp::Params p = {0};
    float *outs[1] = {out};
    return launch_stencil3<AspectOp, XRS_CFG_ASPECT>(in, in_pitch, p, outs, out_pitch, H, W,
                                                           (cudaStream_t)s);
}

int xrs_curvature_f32(const float *in, int64_t in_pitch, float *out, int64_t out_pitch, int64_t H,
                      int64_t W, double cellsize, xrs_stream_t s) {
    const CurvatureOp::Params p = CurvatureOp::Params::make(cellsize);
    float *outs[1] = {out};
    return launch_stencil3<CurvatureOp, XRS_CFG_LIGHT>(in, in_pitch, p, outs, out_pitch, H, W,
                                                              (cudaStream_t)s);
}

int xrs_hillshade_f32(const float *in, int64_t in_pitch, float *out, int64_t out_pitch, int64_t H,
                      int64_t W, double azimuth, double angle_altitude, xrs_stream_t s) {
    const HillshadeOp::Params p = HillshadeOp::Params::make(azimuth, angle_altitude);
    float *outs[1] = {out};
    return launch_stencil3<HillshadeOp, XRS_CFG_LIGHT>(in, in_pitch, p, outs, out_pitch, H, W,
                                                              (cudaStream_t)s);
}

int xrs_surface_suite_f32(const float *in, int64_t in_pitch, float *slope_out, float *aspect_out,
                          float *curvature_out, float *hillshade_out, int64_t out_pitch, int64_t H,
                          int64_t W, double cellsize_x, double cellsize_y, double azimuth,
                          double angle_altitude, xrs_stream_t s) {
    SuiteOp::Params p;
    p.slope = SlopeParams::make(cellsize_x, cellsize_y);
    p.curv = CurvatureOp::Params::make((cellsize_x + cellsize_y) / 2);  // curvature.py:234
    p.hill = HillshadeOp::Params::make(azimuth, angle_altitude);
    float *outs[4] = {slope_out, aspect_out, curvature_out, hillshade_out};
    if (p.slope.rxy == 1.0)
        return launch_stencil3<SuiteSqOp, XRS_CFG_SUITE>(in, in_pitch, p, outs, out_pitch, H, W, (cudaStream_t)s);
    return launch_stencil3<SuiteOp, XRS_CFG_SUITE>(in, in_pitch, p, outs, out_pitch, H, W,
                                                          (cudaStream_t)s);
}

int xrs_focal_mean_f32(const float *in, int64_t in_pitch, float *out, int64_t out_pitch, int64_t H,
                       int64_t W, const double *excludes, int n_ex, xrs_stream_t s) {
    return focal_mean_impl<float, float, XRS_CFG_LIGHT>(in, in_pitch, out, out_pitch, H, W, excludes, n_ex, s);
}
int xrs_focal_mean_f64(const double *in, int64_t in_pitch, double *out, int64_t out_pitch, int64_t H,
                       int64_t W, const double *excludes, int n_ex, xrs_stream_t s) {
    return focal_mean_impl<double, double, XRS_CFG_F64>(in, in_pitch, out, out_pitch, H, W, excludes,
                                                                 n_ex, s);
}
int xrs_focal_mean_f32_f64(const float *in, int64_t in_pitch, double *out, int64_t out_pitch, int64_t H,
                           int64_t W, const double *excludes, int n_ex, xrs_stream_t s) {
    return focal_mean_impl<float, double, XRS_CFG_F32_F64>(in, in_pitch, out, out_pitch, H, W, excludes,
                                                                n_ex, s);
}

}  // extern "C"

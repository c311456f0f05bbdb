// surface.cu -- C-ABI entry points of the 3x3 family (slope, aspect, curvature, hillshade,
// fused suite, focal.mean, 3x3 convolution).  Argument checking lives in stencil3.cuh, launch
// geometry in `geometry` below, and the operator behind each op code in `surface_op`.
#include "surface_ops.cuh"

namespace xrs {

// Pipeline geometry per (operator, source cell type): ROWS rows per TMA stage, STAGES stages, WARPS consumer
// warps per CTA, CTAs per SM (launch_stencil3), swept with scripts/tune/tune5.cu (output in tune5-h100.txt).
struct Geometry {
    int rows, stages, warps, ctas;
};
template <typename Op, typename TS> constexpr Geometry geometry() {
    if constexpr (!std::is_same<TS, typename Op::in_t>::value) {
        // int16 / uint16 / int32 / float64 cells for a float32 operator: 2-byte cells need ROWS % 4 == 0
        // (128-byte aligned boxes); the bytes in flight follow the float32 kernels' sweet spot (~65 KB per SM);
        // the arithmetic-heavy operators get 16 consumer warps, slope two 8-warp CTAs per SM.
        constexpr bool slope = std::is_same<Op, SlopeOp>::value;
        return {sizeof(TS) == 8 ? 2 : 4, sizeof(TS) == 2 ? 4 : 3, slope ? 8 : 16, slope ? 2 : 1};
    }
    // The 4-output suite (~145 registers per thread) keeps the register-store epilogue: its staging does not
    // fit next to an 8 x 2 ring, and the smaller geometries where it fits were not faster with it.
    if (Op::kOutputs == 4) return {8, 2, 12, 1};
    // float64 output (focal.mean f64 and f32 -> f64, 12-16 B per cell)
    if (sizeof(typename Op::out_t) == 8) return {2, 4, 16, 1};
    // With the bulk-store epilogue every single-output float32 operator is fastest, or within 0.3 % of it, at
    // one 16-warp CTA per SM with a 4 x 3 ring (100 KB of input in flight plus 64 KB of output staging).  On an
    // H100 80GB HBM3 (700 W limit), 32768^2, with the loads' evict_last hint, these kernels move 0.84-0.85 of the
    // 3.35 TB/s data sheet, 0.93-0.94 of the card's measured cudaMemcpy rate (3039-3046 GB/s); focal.mean f64
    // above moves 0.88 / 0.97.
    return {4, 3, 16, 1};
}

template <typename Op, typename TS = typename Op::in_t>
static int launch3(const void *in, int64_t in_pitch, const typename Op::Params &p, typename Op::out_t *const *outs,
                   int64_t out_pitch, int64_t H, int64_t W, cudaStream_t s) {
    constexpr Geometry g = geometry<Op, TS>();
    return launch_stencil3<Op, g.rows, g.stages, g.warps, g.ctas, TS>(static_cast<const TS *>(in), in_pitch, p, outs,
                                                                      out_pitch, H, W, s);
}

// Op on a raster of in_dtype cells (OpF32 on float32 cells): float32 as they are, the others converted in
// registers with astype's rounding (int -> f32 and f64 -> f32, round to nearest even), which the reference does
// as a separate `data.astype(np.float32)` pass (slope.py:58,150).
template <typename Op, typename OpF32 = Op>
static int on_cells(int in_dtype, const void *in, int64_t in_pitch, const typename Op::Params &p, float *out,
                    int64_t out_pitch, int64_t H, int64_t W, cudaStream_t s) {
    float *outs[1] = {out};
    switch (in_dtype) {
        case XRS_F32: return launch3<OpF32>(in, in_pitch, p, outs, out_pitch, H, W, s);
        case XRS_I16: return launch3<Op, short>(in, in_pitch, p, outs, out_pitch, H, W, s);
        case XRS_U16: return launch3<Op, unsigned short>(in, in_pitch, p, outs, out_pitch, H, W, s);
        case XRS_I32: return launch3<Op, int>(in, in_pitch, p, outs, out_pitch, H, W, s);
        case XRS_F64: return launch3<Op, double>(in, in_pitch, p, outs, out_pitch, H, W, s);
    }
    set_error("slope, aspect, curvature and hillshade read float32, int16, uint16, int32 or float64 cells");
    return XRS_EUNSUPPORTED;
}

int surface_op(int op, const void *in, int in_dtype, int64_t in_pitch, float *out, int64_t out_pitch, int64_t H,
               int64_t W, const double *p, cudaStream_t s) {
    switch (op) {
        case XRS_OP_SLOPE: {
            XRS_REQUIRE(p != nullptr, "cell sizes missing");
            const SlopeParams q = SlopeParams::make(p[0], p[1]);
            if (q.rxy == 1.0)  // square float32 cells: same arithmetic minus the multiplication by 1
                return on_cells<SlopeOp, SlopeSqOp>(in_dtype, in, in_pitch, q, out, out_pitch, H, W, s);
            return on_cells<SlopeOp>(in_dtype, in, in_pitch, q, out, out_pitch, H, W, s);
        }
        case XRS_OP_ASPECT: return on_cells<AspectOp>(in_dtype, in, in_pitch, {0}, out, out_pitch, H, W, s);
        case XRS_OP_CURVATURE:
            XRS_REQUIRE(p != nullptr, "cell size missing");
            return on_cells<CurvatureOp>(in_dtype, in, in_pitch, CurvatureOp::Params::make(p[0]), out, out_pitch, H,
                                         W, s);
        case XRS_OP_HILLSHADE:
            XRS_REQUIRE(p != nullptr, "azimuth / altitude missing");
            return on_cells<HillshadeOp>(in_dtype, in, in_pitch, HillshadeOp::Params::make(p[0], p[1]), out,
                                         out_pitch, H, W, s);
    }
    set_error("op %d is not slope, aspect, curvature or hillshade", op);
    return XRS_EINVAL;
}

template <typename T, typename TOUT>
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
    if (p.n_ex > 0 || !p.ex_nan) return launch3<OpEx>(in, in_pitch, p, outs, out_pitch, H, W, (cudaStream_t)s);
    typename Op::Params q;
    memcpy(&q, &p, sizeof(q));
    return launch3<Op>(in, in_pitch, q, outs, out_pitch, H, W, (cudaStream_t)s);
}

}  // namespace xrs

using namespace xrs;

// 3x3 kernels of convolve_2d take the warp-strip path (called from conv.cu)
int xrs_conv3_strip(const float *in, int64_t in_pitch, float *out, int64_t out_pitch, int64_t H, int64_t W,
                    const double *kernel, cudaStream_t s) {
    Conv3Op::Params p;
    for (int i = 0; i < 9; ++i) p.w[i] = kernel[i];
    float *outs[1] = {out};
    return launch3<Conv3Op>(in, in_pitch, p, outs, out_pitch, H, W, s);
}

extern "C" {

int xrs_slope_f32(const float *in, int64_t in_pitch, float *out, int64_t out_pitch, int64_t H, int64_t W,
                  double cellsize_x, double cellsize_y, xrs_stream_t s) {
    const double p[2] = {cellsize_x, cellsize_y};
    return surface_op(XRS_OP_SLOPE, in, XRS_F32, in_pitch, out, out_pitch, H, W, p, (cudaStream_t)s);
}

int xrs_aspect_f32(const float *in, int64_t in_pitch, float *out, int64_t out_pitch, int64_t H, int64_t W,
                   xrs_stream_t s) {
    return surface_op(XRS_OP_ASPECT, in, XRS_F32, in_pitch, out, out_pitch, H, W, nullptr, (cudaStream_t)s);
}

int xrs_curvature_f32(const float *in, int64_t in_pitch, float *out, int64_t out_pitch, int64_t H,
                      int64_t W, double cellsize, xrs_stream_t s) {
    return surface_op(XRS_OP_CURVATURE, in, XRS_F32, in_pitch, out, out_pitch, H, W, &cellsize, (cudaStream_t)s);
}

int xrs_hillshade_f32(const float *in, int64_t in_pitch, float *out, int64_t out_pitch, int64_t H,
                      int64_t W, double azimuth, double angle_altitude, xrs_stream_t s) {
    const double p[2] = {azimuth, angle_altitude};
    return surface_op(XRS_OP_HILLSHADE, in, XRS_F32, in_pitch, out, out_pitch, H, W, p, (cudaStream_t)s);
}

// float32 rasters take the entry points above
int xrs_surface_typed(int op, const void *in, int in_dtype, int64_t in_pitch, float *out, int64_t out_pitch,
                      int64_t H, int64_t W, const double *p, xrs_stream_t s) {
    if (H <= 0 || W <= 0) return XRS_OK;
    if (in_dtype == XRS_F32) {
        set_error("direct ingest supports int16, uint16, int32 and float64 rasters");
        return XRS_EUNSUPPORTED;
    }
    return surface_op(op, in, in_dtype, in_pitch, out, out_pitch, H, W, p, (cudaStream_t)s);
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
    if (p.slope.rxy == 1.0) return launch3<SuiteSqOp>(in, in_pitch, p, outs, out_pitch, H, W, (cudaStream_t)s);
    return launch3<SuiteOp>(in, in_pitch, p, outs, out_pitch, H, W, (cudaStream_t)s);
}

int xrs_focal_mean_f32(const float *in, int64_t in_pitch, float *out, int64_t out_pitch, int64_t H,
                       int64_t W, const double *excludes, int n_ex, xrs_stream_t s) {
    return focal_mean_impl(in, in_pitch, out, out_pitch, H, W, excludes, n_ex, s);
}
int xrs_focal_mean_f64(const double *in, int64_t in_pitch, double *out, int64_t out_pitch, int64_t H,
                       int64_t W, const double *excludes, int n_ex, xrs_stream_t s) {
    return focal_mean_impl(in, in_pitch, out, out_pitch, H, W, excludes, n_ex, s);
}
int xrs_focal_mean_f32_f64(const float *in, int64_t in_pitch, double *out, int64_t out_pitch, int64_t H,
                           int64_t W, const double *excludes, int n_ex, xrs_stream_t s) {
    return focal_mean_impl(in, in_pitch, out, out_pitch, H, W, excludes, n_ex, s);
}

}  // extern "C"

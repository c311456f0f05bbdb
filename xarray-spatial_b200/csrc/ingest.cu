// ingest.cu -- slope / aspect / curvature / hillshade reading int16 / uint16 / int32 / float64
// rasters DIRECTLY (SURVEY.md section 8f rank 4).  The reference casts every input to float32 first
// (`data.astype(np.float32)`, slope.py:58,150) -- an extra full pass over the raster; here the
// CTA-wide TMA pipeline of stencil3.cuh moves the raw elements and the consumer lanes widen / narrow
// them to float32 in registers (same rounding as astype: int -> f32 and f64 -> f32, round to nearest
// even), then run the unchanged float32 operators.  For integer rasters the TMA unit can only
// zero-fill out-of-raster cells, so the loader substitutes NaN from the cell coordinates.
#include <type_traits>

#include "surface_ops.cuh"

namespace xrs {

// The CTA-wide TMA pipeline of stencil3.cuh with a source element type TS != float: the ring holds the raw
// cells (32-byte halos, as for float32: 16 cells of 2 bytes, 8 of int32, 4 of float64), consumer lanes convert.
template <typename Op, typename TS, int ROWS, int STAGES, int WARPS, int CTAS>
static int launch_ingest(const void *in, int64_t in_pitch, const typename Op::Params &prm, float *out,
                         int64_t out_pitch, int64_t H, int64_t W, cudaStream_t stream) {
    static_assert(std::is_same<typename Op::in_t, float>::value, "ingest feeds float32 operators");
    CUtensorMap tmap;
    const bool out_aligned = out_pitch % 16 == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0;
    if (!strip_tma_map(&tmap, static_cast<const TS *>(in), in_pitch, H, W, ROWS, out_aligned)) {
        set_error("raster layout not supported by the direct-ingest path (needs 16-byte aligned rows, W %% 4 == 0)");
        return XRS_EUNSUPPORTED;
    }
    OutPtrs<Op> outs;
    outs.p[0] = out;
    outs.pitch_elems = out_pitch / 4;
    return launch_tma<Op, ROWS, STAGES, WARPS, CTAS, TS>(tmap, prm, outs, H, W, stream, kIngestTma);
}

// ring geometry: 2-byte cells need ROWS % 4 == 0 (128-byte aligned boxes); bytes in flight follow the
// float32 kernels' sweet spot (~65 KB per SM), arithmetic-heavy operators get 16 consumer warps
template <typename Op> struct IngestCfg { static constexpr int kWarps = 16, kCtas = 1; };
template <> struct IngestCfg<SlopeOp> { static constexpr int kWarps = 8, kCtas = 2; };

template <typename Op>
static int dispatch_dtype(const void *in, int dtype, int64_t in_pitch, const typename Op::Params &prm, float *out,
                          int64_t out_pitch, int64_t H, int64_t W, cudaStream_t st) {
    constexpr int W_ = IngestCfg<Op>::kWarps, C_ = IngestCfg<Op>::kCtas;
    switch (dtype) {
        case XRS_I16: return launch_ingest<Op, short, 4, 4, W_, C_>(in, in_pitch, prm, out, out_pitch, H, W, st);
        case XRS_U16: return launch_ingest<Op, unsigned short, 4, 4, W_, C_>(in, in_pitch, prm, out, out_pitch, H, W, st);
        case XRS_I32: return launch_ingest<Op, int, 4, 3, W_, C_>(in, in_pitch, prm, out, out_pitch, H, W, st);
        case XRS_F64: return launch_ingest<Op, double, 2, 3, W_, C_>(in, in_pitch, prm, out, out_pitch, H, W, st);
    }
    set_error("direct ingest supports int16, uint16, int32 and float64 rasters");
    return XRS_EUNSUPPORTED;
}

}  // namespace xrs

using namespace xrs;

extern "C" int xrs_surface_typed(int op, const void *in, int in_dtype, int64_t in_pitch, float *out,
                                 int64_t out_pitch, int64_t H, int64_t W, const double *p, xrs_stream_t s) {
    if (H <= 0 || W <= 0) return XRS_OK;
    XRS_REQUIRE(in && out, "NULL pointer");
    XRS_REQUIRE(H < (1LL << 31) - 8 && W < (1LL << 31) - 256, "raster dimension too large");
    cudaStream_t st = (cudaStream_t)s;
    switch (op) {
        case XRS_OP_SLOPE: {
            XRS_REQUIRE(p != nullptr, "cell sizes missing");
            return dispatch_dtype<SlopeOp>(in, in_dtype, in_pitch, SlopeParams::make(p[0], p[1]), out, out_pitch, H,
                                           W, st);
        }
        case XRS_OP_ASPECT: {
            AspectOp::Params q = {0};
            return dispatch_dtype<AspectOp>(in, in_dtype, in_pitch, q, out, out_pitch, H, W, st);
        }
        case XRS_OP_CURVATURE: {
            XRS_REQUIRE(p != nullptr, "cell size missing");
            return dispatch_dtype<CurvatureOp>(in, in_dtype, in_pitch, CurvatureOp::Params::make(p[0]), out,
                                               out_pitch, H, W, st);
        }
        case XRS_OP_HILLSHADE: {
            XRS_REQUIRE(p != nullptr, "azimuth / altitude missing");
            return dispatch_dtype<HillshadeOp>(in, in_dtype, in_pitch, HillshadeOp::Params::make(p[0], p[1]), out,
                                               out_pitch, H, W, st);
        }
    }
    set_error("xrs_surface_typed serves slope, aspect, curvature and hillshade");
    return XRS_EINVAL;
}

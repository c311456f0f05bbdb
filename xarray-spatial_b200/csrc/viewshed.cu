// viewshed.cu -- viewshed (viewshed.py:1122-1502) as a per-cell line-of-sight test (viewshed_los.cuh): a node
// pass writes every cell's angles and gradients to a float64 table, a visibility pass walks each target's ray over
// that table.  Built with -fmad=false like the rest of the library, so the arithmetic is the reference's
// operation order and equals the g++ build of the header bit for bit (DESIGN.md section 4.8).
#include <math.h>

#include "common.cuh"
#include "viewshed_los.cuh"

namespace xrs {
namespace {

using namespace vs;

constexpr int kTile = 16;   // the visibility pass gives each 16 x 16 block a tile of targets with similar rays

template <typename T> __global__ void vs_node_kernel(View v, Cells<T> z, Node *nodes) {
    const int64_t n = v.H * v.W;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = k / v.W, c = k - r * v.W;
        if (r == v.vr && c == v.vc) continue;   // the observer has no node
        nodes[k] = make_node(v, [&](int64_t rr, int64_t cc) { return (double)z(rr, cc); }, r, c);
    }
}

__global__ void __launch_bounds__(kTile * kTile) vs_visibility_kernel(View v, const Node *__restrict__ nodes,
                                                                      double *out, int64_t out_pitch) {
    const int64_t r = (int64_t)blockIdx.y * kTile + threadIdx.y, c = (int64_t)blockIdx.x * kTile + threadIdx.x;
    if (r >= v.H || c >= v.W) return;
    const int64_t W = v.W;
    out[r * out_pitch + c] = cell_value(v, [&](int64_t rr, int64_t cc) { return nodes[rr * W + cc]; }, r, c);
}

int64_t scratch_need(int64_t H, int64_t W) { return H * W * (int64_t)sizeof(Node); }

int check_shape(int64_t H, int64_t W) {
    XRS_REQUIRE(H >= 0 && W >= 0, "negative raster shape");
    XRS_REQUIRE(H < INT32_MAX && W < INT32_MAX, "rows and columns must each be below 2^31");
    if (H > 0 && W > 0 && H > (INT64_MAX / (int64_t)sizeof(Node)) / W) {
        set_error("a %lld x %lld raster's node table does not fit in 64-bit sizes", (long long)H, (long long)W);
        return XRS_ENOMEM;
    }
    return XRS_OK;
}

template <typename T> int run(const View &v, const void *in, int64_t in_pitch, double *out, int64_t out_pitch,
                              Node *nodes, cudaStream_t s) {
    int64_t g = (v.H * v.W + 255) / 256;
    if (g > 65536) g = 65536;
    vs_node_kernel<T><<<(unsigned)g, 256, 0, s>>>(v, Cells<T>{(const char *)in, in_pitch}, nodes);
    XRS_CUDA(cudaGetLastError());
    const dim3 grid((unsigned)((v.W + kTile - 1) / kTile), (unsigned)((v.H + kTile - 1) / kTile));
    vs_visibility_kernel<<<grid, dim3(kTile, kTile), 0, s>>>(v, nodes, out, out_pitch / 8);
    XRS_CUDA(cudaGetLastError());
    return XRS_OK;
}

}  // namespace
}  // namespace xrs

using namespace xrs;

extern "C" int xrs_viewshed_scratch_bytes(int64_t H, int64_t W, int64_t *bytes) {
    XRS_REQUIRE(bytes != nullptr, "NULL pointer");
    const int rc = check_shape(H, W);
    if (rc) return rc;
    *bytes = scratch_need(H, W);
    return XRS_OK;
}

extern "C" int xrs_viewshed(const void *in, int in_dtype, int64_t in_pitch, int64_t H, int64_t W, int64_t vp_row,
                            int64_t vp_col, double vp_elev, double target_elev, double ew_res, double ns_res,
                            double *out, int64_t out_pitch, void *scratch, int64_t scratch_bytes, xrs_stream_t s) {
    int rc = check_shape(H, W);
    if (rc) return rc;
    XRS_REQUIRE(H > 0 && W > 0, "viewshed needs a raster of at least one cell");
    XRS_REQUIRE(vp_row >= 0 && vp_row < H && vp_col >= 0 && vp_col < W, "observer outside the raster");
    XRS_REQUIRE(in && out, "NULL pointer");
    XRS_TRY(check_cells_arg(in, in_dtype, kRasterCells, in_pitch, W));
    XRS_TRY(check_out_pitch(out_pitch, 8, W));
    XRS_TRY(check_scratch(scratch, scratch_bytes, scratch_need(H, W), "xrs_viewshed_scratch_bytes"));
    const View v{H, W, vp_row, vp_col, vp_elev, target_elev, ew_res, ns_res};
    return with_cell_type(kRasterCells, in_dtype, [&](auto z) {
        return run<decltype(z)>(v, in, in_pitch, out, out_pitch, (Node *)scratch, (cudaStream_t)s);
    });
}

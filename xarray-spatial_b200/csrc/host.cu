// host.cu -- host-buffer (end-to-end) entry point: the same operators on HOST rasters.
//
// This is what a numpy-backed DataArray call binds (the reference's `_run_numpy` slot,
// e.g. slope.py:79).  The raster is cut into row chunks of ~32 MiB; chunk c is copied
// host->device on a copy stream while chunk c-1 is computed and chunk c-2 travels back,
// using three device slots and events, so PCIe runs full duplex and the kernels hide behind
// it.  Each chunk carries `r` halo rows above and below (r = kernel radius); the operator
// treats the chunk view as a raster of its own, so its first/last r output rows are only
// correct when they coincide with the real raster edge -- interior halo rows are simply
// not copied back.  Host buffers may be pageable (works, slower) or pinned (xrs_host_alloc).
//
// Several GPUs (the `devices` list of xrs_host_stencil): the output rows are cut into one stripe per
// device and every device runs the pipeline above on its stripe from its own host thread -- one PCIe
// link each, no device-to-device traffic at all, because a stripe's halo rows come straight from the
// host raster like any chunk's.  This is the reference's `dask.map_overlap(depth=r)` over row
// blocks (slope.py:94-97) with the blocks being PCIe-sized.
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "common.cuh"

namespace xrs {

struct Slot {
    void *din = nullptr, *dout = nullptr;
    size_t cap_in = 0, cap_out = 0;
    cudaEvent_t in_done = nullptr, k_done = nullptr, out_done = nullptr;
};
struct HostCtx {
    bool init = false;
    cudaStream_t s_in = nullptr, s_k = nullptr, s_out = nullptr;
    Slot slot[3];
    std::mutex mu;
};
static HostCtx g_ctx[16];

static int ensure_ctx(HostCtx &c) {
    if (c.init) return XRS_OK;
    XRS_CUDA(cudaStreamCreateWithFlags(&c.s_in, cudaStreamNonBlocking));
    XRS_CUDA(cudaStreamCreateWithFlags(&c.s_k, cudaStreamNonBlocking));
    XRS_CUDA(cudaStreamCreateWithFlags(&c.s_out, cudaStreamNonBlocking));
    for (auto &s : c.slot) {
        XRS_CUDA(cudaEventCreateWithFlags(&s.in_done, cudaEventDisableTiming));
        XRS_CUDA(cudaEventCreateWithFlags(&s.k_done, cudaEventDisableTiming));
        XRS_CUDA(cudaEventCreateWithFlags(&s.out_done, cudaEventDisableTiming));
    }
    c.init = true;
    return XRS_OK;
}
static int ensure_cap(void **p, size_t *cap, size_t need) {
    if (*cap >= need) return XRS_OK;
    if (*p) XRS_CUDA(cudaFree(*p));
    *p = nullptr;
    *cap = 0;
    XRS_CUDA(cudaMalloc(p, need));
    *cap = need;
    return XRS_OK;
}

// The cell sizes and halo of a host request.  host_op_shape is the one place that decides them and
// checks the request, before any CUDA call:
//   op                                   in_dtype                                        out
//   SLOPE, ASPECT, CURVATURE, HILLSHADE  F32; F64, I32, I16, U16 when W % 4 == 0         float32
//   FOCAL_MEAN                           F32, F64                                        float64
//   CONVOLVE, FOCAL_STAT                 F32                                             float32
struct OpShape {
    int in_size, out_size, radius;
};

static int host_op_shape(int op, int in_dtype, const double *p, const double *aux, int64_t W, OpShape *sh) {
    sh->in_size = (in_dtype == XRS_F64) ? 8 : (in_dtype == XRS_I16 || in_dtype == XRS_U16) ? 2 : 4;
    sh->out_size = 4;
    sh->radius = 1;
    switch (op) {
        case XRS_OP_SLOPE:
        case XRS_OP_ASPECT:
        case XRS_OP_CURVATURE:
        case XRS_OP_HILLSHADE:
            XRS_REQUIRE(p || op == XRS_OP_ASPECT, "scalar parameters missing");
            if (in_dtype == XRS_F32) return XRS_OK;
            // raw cells go to the direct-ingest TMA kernels (surface_op), which need W % 4 == 0
            XRS_REQUIRE(in_dtype == XRS_F64 || in_dtype == XRS_I32 || in_dtype == XRS_I16 || in_dtype == XRS_U16,
                        "in_dtype must be float32, int16, uint16, int32 or float64");
            XRS_REQUIRE(W % 4 == 0, "int16 / uint16 / int32 / float64 host input needs W % 4 == 0");
            return XRS_OK;
        case XRS_OP_FOCAL_MEAN:  // float64 out: focal.mean's `astype(float)` (focal.py:257)
            XRS_REQUIRE(in_dtype == XRS_F32 || in_dtype == XRS_F64, "focal mean takes float32 or float64 cells");
            sh->out_size = 8;
            return XRS_OK;
        case XRS_OP_CONVOLVE:
        case XRS_OP_FOCAL_STAT:
            XRS_REQUIRE(in_dtype == XRS_F32, "convolve and focal statistics take float32 cells");
            XRS_REQUIRE(p && aux, "kernel parameters missing");
            if (const int rc = check_window((int)p[0], (int)p[1])) return rc;
            sh->radius = (int)p[0] / 2;
            return XRS_OK;
    }
    set_error("unknown op %d", op);
    return XRS_EINVAL;
}

static int run_op(int op, int in_dtype, const void *din, void *dout, int64_t pitch, int64_t opitch, int64_t h,
                  int64_t W, const double *p, const double *aux, int naux, cudaStream_t s) {
    const float *fi = (const float *)din;
    float *fo = (float *)dout;
    switch (op) {
        case XRS_OP_SLOPE:
        case XRS_OP_ASPECT:
        case XRS_OP_CURVATURE:
        case XRS_OP_HILLSHADE: return surface_op(op, din, in_dtype, pitch, fo, opitch, h, W, p, s);
        case XRS_OP_FOCAL_MEAN:
            if (in_dtype == XRS_F64)
                return xrs_focal_mean_f64((const double *)din, pitch, (double *)dout, opitch, h, W, aux, naux, s);
            return xrs_focal_mean_f32_f64(fi, pitch, (double *)dout, opitch, h, W, aux, naux, s);
        case XRS_OP_CONVOLVE: return xrs_convolve2d_f32(fi, pitch, fo, opitch, h, W, aux, (int)p[0], (int)p[1], s);
        case XRS_OP_FOCAL_STAT:
            return xrs_focal_stat_f32(fi, pitch, fo, opitch, h, W, aux, (int)p[0], (int)p[1], (int)p[2], s);
    }
    set_error("unknown op %d", op);
    return XRS_EINVAL;
}

}  // namespace xrs

using namespace xrs;

// Output rows [y_begin, y_end) of the H x W raster on `device`; the request was checked by host_op_shape.
static int host_pipeline(int op, int in_dtype, const OpShape &sh, const void *in, void *out, int64_t H, int64_t W,
                         const double *p, const double *aux, int naux, int device, int64_t y_begin, int64_t y_end) {
    const int radius = sh.radius;
    int prev = 0;
    XRS_CUDA(cudaGetDevice(&prev));
    XRS_CUDA(cudaSetDevice(device));
    HostCtx &c = g_ctx[device];
    std::lock_guard<std::mutex> lock(c.mu);
    int rc = ensure_ctx(c);
    if (rc) { cudaSetDevice(prev); return rc; }

    // device row pitch: multiple of 16 bytes so the TMA kernels apply whenever W % 4 == 0
    const int64_t row_bytes = W * sh.in_size, orow_bytes = W * sh.out_size;
    const int64_t pitch = (row_bytes + 15) / 16 * 16, opitch = (orow_bytes + 15) / 16 * 16;
    const int64_t span = y_end - y_begin;
    int64_t rows = (32LL << 20) / pitch;
    if (rows < 8 * radius + 8) rows = 8 * radius + 8;
    if (rows > span) rows = span;
    const int64_t n_chunks = (span + rows - 1) / rows;
    const size_t cap = (size_t)(rows + 2 * radius) * pitch, ocap = (size_t)(rows + 2 * radius) * opitch;

    for (int64_t ci = 0; ci < n_chunks && rc == XRS_OK; ++ci) {
        Slot &s = c.slot[ci % 3];
        const int64_t r0 = y_begin + ci * rows, r1 = (r0 + rows < y_end) ? r0 + rows : y_end;
        const int64_t a0 = (r0 - radius > 0) ? r0 - radius : 0, a1 = (r1 + radius < H) ? r1 + radius : H;
        const int64_t h = a1 - a0;
        // the slot is free once its previous D2H has finished
        cudaError_t e = cudaEventSynchronize(s.out_done);
        if (e != cudaSuccess) { rc = cuda_fail(e, "cudaEventSynchronize"); break; }
        rc = ensure_cap(&s.din, &s.cap_in, cap);
        if (rc) break;
        rc = ensure_cap(&s.dout, &s.cap_out, ocap);
        if (rc) break;
        e = cudaMemcpy2DAsync(s.din, pitch, (const char *)in + a0 * row_bytes, row_bytes, row_bytes, h,
                              cudaMemcpyHostToDevice, c.s_in);
        if (e == cudaSuccess) e = cudaEventRecord(s.in_done, c.s_in);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(c.s_k, s.in_done, 0);
        if (e != cudaSuccess) { rc = cuda_fail(e, "H2D enqueue"); break; }
        rc = run_op(op, in_dtype, s.din, s.dout, pitch, opitch, h, W, p, aux, naux, c.s_k);
        if (rc) break;
        e = cudaEventRecord(s.k_done, c.s_k);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(c.s_out, s.k_done, 0);
        if (e == cudaSuccess)
            e = cudaMemcpy2DAsync((char *)out + r0 * orow_bytes, orow_bytes,
                                  (const char *)s.dout + (r0 - a0) * opitch, opitch, orow_bytes, r1 - r0,
                                  cudaMemcpyDeviceToHost, c.s_out);
        if (e == cudaSuccess) e = cudaEventRecord(s.out_done, c.s_out);
        if (e != cudaSuccess) { rc = cuda_fail(e, "D2H enqueue"); break; }
    }
    cudaError_t e = cudaStreamSynchronize(c.s_out);
    cudaError_t e2 = cudaStreamSynchronize(c.s_k);
    cudaError_t e3 = cudaStreamSynchronize(c.s_in);
    if (rc == XRS_OK && (e != cudaSuccess || e2 != cudaSuccess || e3 != cudaSuccess))
        rc = cuda_fail(e != cudaSuccess ? e : (e2 != cudaSuccess ? e2 : e3), "pipeline synchronize");
    cudaSetDevice(prev);
    return rc;
}

// Row stripes over several devices, one host thread and one PCIe link per device.  Errors: the
// first failing stripe's status and message are returned (the message is copied out of the worker
// thread, whose thread-local error string the caller cannot see).
extern "C" int xrs_host_stencil(int op, const void *in, int in_dtype, void *out, int64_t H, int64_t W,
                                const double *p, const double *aux, int naux, const int *devices, int n_devices) {
    XRS_REQUIRE(devices != nullptr && n_devices >= 1 && n_devices <= 16, "1 .. 16 devices expected");
    for (int i = 0; i < n_devices; ++i) {
        XRS_REQUIRE(devices[i] >= 0 && devices[i] < 16, "device index out of range");
        for (int j = 0; j < i; ++j) XRS_REQUIRE(devices[i] != devices[j], "device listed twice");
    }
    OpShape sh;
    const int bad = host_op_shape(op, in_dtype, p, aux, W, &sh);
    if (bad) return bad;
    if (H <= 0 || W <= 0) return XRS_OK;
    XRS_REQUIRE(in && out, "NULL host pointer");
    // stripes shorter than a few halos are not worth a device
    int n = n_devices;
    while (n > 1 && H / n < 8 * sh.radius + 8) --n;
    if (n == 1) return host_pipeline(op, in_dtype, sh, in, out, H, W, p, aux, naux, devices[0], 0, H);
    std::vector<int> rc(n, XRS_OK);
    std::vector<std::string> msg(n);
    std::vector<std::thread> th;
    const int64_t base = H / n, rem = H % n;
    int64_t y = 0;
    for (int i = 0; i < n; ++i) {
        const int64_t h = base + (i < rem ? 1 : 0);
        const int64_t y0 = y, y1 = y + h;
        y = y1;
        th.emplace_back([&, i, y0, y1] {
            rc[i] = host_pipeline(op, in_dtype, sh, in, out, H, W, p, aux, naux, devices[i], y0, y1);
            if (rc[i] != XRS_OK) msg[i] = xrs_last_error_string();
        });
    }
    for (auto &t : th) t.join();
    for (int i = 0; i < n; ++i)
        if (rc[i] != XRS_OK) {
            set_error("device %d: %s", devices[i], msg[i].c_str());
            return rc[i];
        }
    return XRS_OK;
}

// release the per-device staging buffers (tests / interpreter shutdown)
extern "C" int xrs_host_release(int device) {
    XRS_REQUIRE(device >= 0 && device < 16, "device index out of range");
    HostCtx &c = g_ctx[device];
    std::lock_guard<std::mutex> lock(c.mu);
    if (!c.init) return XRS_OK;
    int prev = 0;
    cudaGetDevice(&prev);
    cudaSetDevice(device);
    for (auto &s : c.slot) {
        if (s.din) cudaFree(s.din);
        if (s.dout) cudaFree(s.dout);
        s.din = s.dout = nullptr;
        s.cap_in = s.cap_out = 0;
    }
    cudaSetDevice(prev);
    return XRS_OK;
}

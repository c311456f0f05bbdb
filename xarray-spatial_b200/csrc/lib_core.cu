// lib_core.cu -- error state, device properties, tensor-map encoding, pinned memory.
#include <stdarg.h>

#include "stencil3.cuh"

namespace xrs {

static thread_local char g_err[512] = "";

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int cuda_fail(cudaError_t e, const char *what) {
    set_error("CUDA error %d (%s) in %s", (int)e, cudaGetErrorString(e), what);
    return XRS_ECUDA;
}

int sm_count(int device) {
    static int cache[64];
    if (device < 0 && cudaGetDevice(&device) != cudaSuccess) return 132;   // an H100 SXM
    if (device < 0 || device >= 64) return 132;
    if (cache[device] == 0) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || n <= 0)
            n = 132;
        cache[device] = n;
    }
    return cache[device];
}

LaunchInfo &last_launch_info() {
    static thread_local LaunchInfo li = {0, 0, 0, 0};
    return li;
}

typedef CUresult (*encode_tiled_fn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *,
                                    const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
                                    const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static encode_tiled_fn get_encode_fn() {
    static encode_tiled_fn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void *p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        // resolved through the runtime so libcuda is not a link-time dependency
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<encode_tiled_fn>(p);
    }
    return fn;
}

bool make_tensor_map_2d(CUtensorMap *map, const void *base, int64_t pitch_bytes, int64_t H, int64_t W,
                        xrs_dtype dtype, int box_w, int box_h) {
    CUtensorMapDataType dt;
    int esz;
    switch (dtype) {
        case XRS_F32: dt = CU_TENSOR_MAP_DATA_TYPE_FLOAT32; esz = 4; break;
        case XRS_F64: dt = CU_TENSOR_MAP_DATA_TYPE_FLOAT64; esz = 8; break;
        case XRS_I32: dt = CU_TENSOR_MAP_DATA_TYPE_INT32; esz = 4; break;
        case XRS_I16: case XRS_U16: dt = CU_TENSOR_MAP_DATA_TYPE_UINT16; esz = 2; break;
        default: return false;
    }
    if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || pitch_bytes % 16 != 0) return false;
    if ((int64_t)box_w * esz % 16 != 0 || box_w > 256 || box_h > 256) return false;
    encode_tiled_fn fn = get_encode_fn();
    if (!fn) return false;
    const cuuint64_t dims[2] = {(cuuint64_t)W, (cuuint64_t)H};
    const cuuint64_t strides[1] = {(cuuint64_t)pitch_bytes};
    const cuuint32_t box[2] = {(cuuint32_t)box_w, (cuuint32_t)box_h};
    const cuuint32_t estr[2] = {1, 1};
    const CUtensorMapFloatOOBfill fill = (dtype == XRS_F32 || dtype == XRS_F64)
                                             ? CU_TENSOR_MAP_FLOAT_OOB_FILL_NAN_REQUEST_ZERO_FMA
                                             : CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE;
    return fn(map, dt, 2, const_cast<void *>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
              CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, fill) == CUDA_SUCCESS;
}

int resident_ctas(const void *kernel, int threads, size_t smem, int max_per_sm, int64_t *resident) {
    XRS_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    XRS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem));
    if (per_sm > max_per_sm) per_sm = max_per_sm;
    if (per_sm < 1) per_sm = 1;
    *resident = (int64_t)sm_count() * per_sm;
    return XRS_OK;
}

}  // namespace xrs

extern "C" {

int xrs_abi_version(void) { return XRS_ABI_VERSION; }
const char *xrs_last_error_string(void) { return xrs::g_err; }

int xrs_device_count(int *n) {
    XRS_REQUIRE(n != nullptr, "n is NULL");
    XRS_CUDA(cudaGetDeviceCount(n));
    return XRS_OK;
}
int xrs_device_sm_count(int device, int *sm) {
    XRS_REQUIRE(sm != nullptr, "sm_count is NULL");
    int n = 0;
    XRS_CUDA(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device));
    *sm = n;
    return XRS_OK;
}
int xrs_host_alloc(void **ptr, int64_t bytes) {
    XRS_REQUIRE(ptr != nullptr && bytes >= 0, "bad arguments");
    XRS_CUDA(cudaHostAlloc(ptr, (size_t)bytes, cudaHostAllocPortable));
    return XRS_OK;
}
int xrs_host_free(void *ptr) {
    XRS_CUDA(cudaFreeHost(ptr));
    return XRS_OK;
}
// test hook: which kernel the last launch on this thread chose (codes in xrs_b200.h)
int xrs_debug_last_used_tma(void) { return xrs::last_launch_info().kind; }
int xrs_debug_last_grid(void) { return xrs::last_launch_info().grid; }
// test hook (host only, no device needed): the row-segment height the persistent kernels would pick
int64_t xrs_debug_pick_seg_rows(int64_t H, int64_t n_tiles, int64_t resident, int64_t min_rows, int64_t lead,
                                int64_t quantum, int64_t want) {
    return xrs::pick_seg_rows(H, n_tiles, resident, min_rows, lead, quantum, want);
}

}  // extern "C"

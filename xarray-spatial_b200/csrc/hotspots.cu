// hotspots.cu -- the two extra pieces focal.hotspots needs beside convolve_2d (focal.py:881-937):
// global NaN-skipping mean / std of the raster (one streaming pass, f64 accumulation) and the
// z-score -> confidence classification epilogue (int8).
#include <math.h>

#include "common.cuh"

namespace xrs {

// partial[0] = count, [1] = sum(v - pivot), [2] = sum((v - pivot)^2), accumulated with atomics
__global__ void __launch_bounds__(256) global_stats_kernel(const float *__restrict__ v, int64_t n, double pivot,
                                                           double *partial) {
    double s1 = 0.0, s2 = 0.0;
    unsigned long long cnt = 0;
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, nt = (int64_t)gridDim.x * blockDim.x;
    const bool al = (reinterpret_cast<uintptr_t>(v) & 15) == 0;
    const int64_t n4 = al ? (n >> 2) : 0;
    for (int64_t i = tid; i < n4; i += nt) {
        const float4 q = __ldcs(reinterpret_cast<const float4 *>(v) + i);
        const float w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const bool ok = (w[k] == w[k]);  // np.nanmean / np.nanstd skip NaN only
            const double d = ok ? (double)w[k] - pivot : 0.0;
            s1 += d;
            s2 = fma(d, d, s2);
            cnt += ok ? 1ull : 0ull;
        }
    }
    for (int64_t i = (n4 << 2) + tid; i < n; i += nt) {
        const float w = v[i];
        if (w == w) { const double d = (double)w - pivot; s1 += d; s2 = fma(d, d, s2); cnt += 1ull; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        s2 += __shfl_xor_sync(0xffffffffu, s2, o);
        cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    }
    if ((threadIdx.x & 31) == 0) {
        atomicAdd(&partial[0], (double)cnt);
        atomicAdd(&partial[1], s1);
        atomicAdd(&partial[2], s2);
    }
}

// focal.py:881-915 `_calc_hotspots_numpy` on z = (mean - global_mean) / global_std in float32.  Numba
// compares the float32 |z| with the float64 literals in float64, so this does too: in float32 the
// threshold 1.96 rounds up to 1.96000003815, and z = 1.96f would be classified 90 instead of 95.
__global__ void __launch_bounds__(256) hotspots_classify_kernel(const float *__restrict__ mean, int64_t n,
                                                                float gmean, float gstd, signed char *out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float z = (mean[i] - gmean) / gstd;
        const double az = fabs((double)z);
        double p = 1.0;
        if (az >= 2.33) p = 0.0099; else if (az >= 1.65) p = 0.0495; else if (az >= 1.29) p = 0.0985;
        int conf = 0;
        if (az > 2.58 && p < 0.01) conf = 99; else if (az > 1.96 && p < 0.05) conf = 95; else if (az > 1.65 && p < 0.1) conf = 90;
        const int hc = z > 0.f ? 1 : (z < 0.f ? -1 : 0);
        out[i] = (signed char)(hc * conf);
    }
}

}  // namespace xrs

using namespace xrs;

extern "C" {

int xrs_global_stats_f32(const float *values, int64_t n, double pivot, double *partial3, xrs_stream_t s) {
    XRS_REQUIRE(partial3 != nullptr && (values != nullptr || n == 0), "NULL pointer");
    XRS_CUDA(cudaMemsetAsync(partial3, 0, 3 * sizeof(double), (cudaStream_t)s));
    if (n <= 0) return XRS_OK;
    int64_t grid = (n / 4 + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 8;
    if (grid > cap) grid = cap;
    if (grid < 1) grid = 1;
    global_stats_kernel<<<(unsigned)grid, 256, 0, (cudaStream_t)s>>>(values, n, pivot, partial3);
    XRS_CUDA(cudaGetLastError());
    return XRS_OK;
}

int xrs_hotspots_classify_f32(const float *mean, int64_t n, double global_mean, double global_std, int8_t *out,
                              xrs_stream_t s) {
    if (n <= 0) return XRS_OK;
    XRS_REQUIRE(mean && out, "NULL pointer");
    int64_t grid = (n + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 8;
    if (grid > cap) grid = cap;
    hotspots_classify_kernel<<<(unsigned)grid, 256, 0, (cudaStream_t)s>>>(mean, n, (float)global_mean, (float)global_std,
                                                                         (signed char *)out);
    XRS_CUDA(cudaGetLastError());
    return XRS_OK;
}

}  // extern "C"

// multispectral.cu -- per-cell band indices (multispectral.py): float4 grid-stride kernels.
// Arithmetic types follow the reference's Numba CPU kernels exactly (which subexpressions are
// float32 and which are promoted to float64), so results are bit-identical to the oracle up to
// the f64 division being replaced by nothing -- divisions are kept as IEEE divisions.
#include "common.cuh"

namespace xrs {

struct NormRatio {  // multispectral.py:825-841 -- pure f32
    __device__ __forceinline__ float operator()(float a, float b, float) const {
        const float den = a + b;
        return den == 0.0f ? __int_as_float(0x7fc00000) : (a - b) / den;
    }
};
// :876-890 -- numerator f32; nir + red + L in the type Numba gives it, which follows L's type: f32 for a float32,
// int8, int16, uint8 or bool L (f32_sum), f64 for a Python float or int and the wider NumPy types; the
// product with 1 + L and the division are f64 either way.
struct Savi {
    double L, onepL;
    int f32_sum;
    __device__ __forceinline__ float operator()(float nir, float red, float) const {
        const float num = nir - red;
        const double soma = f32_sum ? (double)((nir + red) + (float)L) : (double)(nir + red) + L;
        const double den = soma * onepL;
        return den != 0.0 ? (float)((double)num / den) : __int_as_float(0x7fc00000);
    }
};
struct Evi {  // :175-188
    double c1, c2, L, G;
    __device__ __forceinline__ float operator()(float nir, float red, float blue) const {
        const float num = nir - red;
        const double den = (((double)nir + c1 * (double)red) - c2 * (double)blue) + L;
        return den != 0.0 ? (float)(G * ((double)num / den)) : __int_as_float(0x7fc00000);
    }
};
struct Arvi {  // :29-43
    __device__ __forceinline__ float operator()(float nir, float red, float blue) const {
        const double r2 = 2.0 * (double)red;
        const double num = ((double)nir - r2) + (double)blue;
        const double den = ((double)nir + r2) + (double)blue;
        return den != 0.0 ? (float)(num / den) : __int_as_float(0x7fc00000);
    }
};
struct Gci {  // :350-360 -- f32 division, then `- 1` in f64
    __device__ __forceinline__ float operator()(float nir, float green, float) const {
        return green != 0.0f ? (float)((double)(nir / green) - 1.0) : __int_as_float(0x7fc00000);
    }
};
struct Sipi {  // :1017-1030 -- pure f32
    __device__ __forceinline__ float operator()(float nir, float red, float blue) const {
        const float den = nir - red;
        return den != 0.0f ? (nir - blue) / den : __int_as_float(0x7fc00000);
    }
};
struct Ebbi {  // :1160-1173 -- sqrt in f32, 10 * in f64
    __device__ __forceinline__ float operator()(float red, float swir, float tir) const {
        const float num = swir - red;
        const double den = 10.0 * (double)sqrtf(swir + tir);
        return den != 0.0 ? (float)((double)num / den) : __int_as_float(0x7fc00000);
    }
};

template <int NIN, typename F>
__global__ void __launch_bounds__(256) band_kernel(const float *__restrict__ a, const float *__restrict__ b,
                                                   const float *__restrict__ c, float *__restrict__ out,
                                                   int64_t n, int vec, const F f) {
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t nthreads = (int64_t)gridDim.x * blockDim.x;
    if (vec) {
        const int64_t n4 = n >> 2;
        const float4 *a4 = reinterpret_cast<const float4 *>(a);
        const float4 *b4 = reinterpret_cast<const float4 *>(b);
        const float4 *c4 = reinterpret_cast<const float4 *>(c);
        float4 *o4 = reinterpret_cast<float4 *>(out);
        for (int64_t i = tid; i < n4; i += nthreads) {
            const float4 x = __ldcs(a4 + i), y = __ldcs(b4 + i);
            float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
            if (NIN == 3) z = __ldcs(c4 + i);
            __stcs(o4 + i, make_float4(f(x.x, y.x, z.x), f(x.y, y.y, z.y), f(x.z, y.z, z.z), f(x.w, y.w, z.w)));
        }
        for (int64_t i = (n4 << 2) + tid; i < n; i += nthreads) out[i] = f(a[i], b[i], NIN == 3 ? c[i] : 0.f);
    } else {
        for (int64_t i = tid; i < n; i += nthreads) out[i] = f(a[i], b[i], NIN == 3 ? c[i] : 0.f);
    }
}

template <int NIN, typename F>
static int launch_band(const float *a, const float *b, const float *c, float *out, int64_t n, const F &f,
                       xrs_stream_t s) {
    if (n <= 0) return XRS_OK;
    XRS_REQUIRE(a && b && out && (NIN == 2 || c), "NULL band pointer");
    if (NIN == 2) c = a;
    const bool vec = ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) |
                       reinterpret_cast<uintptr_t>(c) | reinterpret_cast<uintptr_t>(out)) & 15) == 0;
    const int64_t work = vec ? (n + 3) / 4 : n;
    band_kernel<NIN, F><<<(unsigned)stride_grid(work), 256, 0, (cudaStream_t)s>>>(a, b, c, out, n, vec ? 1 : 0, f);
    XRS_CUDA(cudaGetLastError());
    return XRS_OK;
}

}  // namespace xrs

using namespace xrs;

extern "C" {
int xrs_normalized_ratio_f32(const float *a, const float *b, float *out, int64_t n, xrs_stream_t s) {
    return launch_band<2>(a, b, nullptr, out, n, NormRatio{}, s);
}
int xrs_savi_f32(const float *nir, const float *red, double soil_factor, int f32_sum, float *out, int64_t n,
                 xrs_stream_t s) {
    return launch_band<2>(nir, red, nullptr, out, n, Savi{soil_factor, 1.0 + soil_factor, f32_sum}, s);
}
int xrs_evi_f32(const float *nir, const float *red, const float *blue, double c1, double c2,
                double soil_factor, double gain, float *out, int64_t n, xrs_stream_t s) {
    return launch_band<3>(nir, red, blue, out, n, Evi{c1, c2, soil_factor, gain}, s);
}
int xrs_arvi_f32(const float *nir, const float *red, const float *blue, float *out, int64_t n,
                 xrs_stream_t s) {
    return launch_band<3>(nir, red, blue, out, n, Arvi{}, s);
}
int xrs_gci_f32(const float *nir, const float *green, float *out, int64_t n, xrs_stream_t s) {
    return launch_band<2>(nir, green, nullptr, out, n, Gci{}, s);
}
int xrs_sipi_f32(const float *nir, const float *red, const float *blue, float *out, int64_t n,
                 xrs_stream_t s) {
    return launch_band<3>(nir, red, blue, out, n, Sipi{}, s);
}
int xrs_ebbi_f32(const float *red, const float *swir, const float *tir, float *out, int64_t n,
                 xrs_stream_t s) {
    return launch_band<3>(red, swir, tir, out, n, Ebbi{}, s);
}
}

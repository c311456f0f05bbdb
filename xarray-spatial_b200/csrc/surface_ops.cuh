// surface_ops.cuh -- per-row operators for the 3x3 skeleton (stencil3.cuh).
//
// Numerics follow the reference's *CPU* kernels, which do the Horn sums in float64 because
// Numba promotes `2 * f32` (SURVEY.md section 0 fact 5): the column differences / weighted row
// sums are formed in f64 (they are EXACT there for any realistic raster: sums of <= 8
// float32 values), so re-associating them row by row changes nothing; the transcendental
// tail (sqrt / atan / atan2) is evaluated in f32 on the correctly-rounded f64 intermediate,
// which keeps the result within ~3e-7 relative of the oracle (bar: 1e-5).
#pragma once
#include <math.h>

#include "stencil3.cuh"

namespace xrs {

// Column difference D[i] = right - left and Horn row sum S[i] = left + 2*mid + right of one
// input row, in f64, for the 4 cells of a lane.
struct HornRow {
    double D[4], S[4];
};
__device__ __forceinline__ HornRow horn_row(const Row6<float> &r) {
    double w[6];
    w[0] = (double)r.l;
#pragma unroll
    for (int i = 0; i < 4; ++i) w[i + 1] = (double)r.c[i];
    w[5] = (double)r.r;
    HornRow h;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        h.D[i] = w[i + 2] - w[i];
        h.S[i] = fma(2.0, w[i + 1], w[i]) + w[i + 2];
    }
    return h;
}

// ------------------------------------------------------------------ slope (slope.py:56-76)
// SQUARE = cellsize_x == cellsize_y (rxy == 1 exactly): the X * rxy multiplication is skipped,
// which changes nothing (X * 1.0 == X) and saves one FP64 instruction per cell.
struct SlopeParams {
    double rxy;  // (1/(8 csx)) / (1/(8 csy)) = csy / csx
    float ky2;   // (1/(8 csy))^2
    static SlopeParams make(double cellsize_x, double cellsize_y) {
        const double kx = 1.0 / (8.0 * cellsize_x), ky = 1.0 / (8.0 * cellsize_y);
        SlopeParams p;
        p.rxy = kx / ky;
        p.ky2 = (float)(ky * ky);
        return p;
    }
};
// p = dz_dx^2 + dz_dy^2 = ky^2 ((X kx/ky)^2 + Y^2): X, Y are exact in f64, the sum of squares
// is formed in f64 and only then rounded to f32 (the result needs f32 accuracy).
template <bool SQUARE> __device__ __forceinline__ float slope_q(double X, double Y, const SlopeParams &p) {
    if constexpr (SQUARE) return (float)fma(X, X, Y * Y);
    const double xs = X * p.rxy;
    return (float)fma(xs, xs, Y * Y);
}
// four cells of one lane: the f32 tail (scale, rsqrt, polynomial)
__device__ __forceinline__ void slope_tail4(const float (&q)[4], float ky2, float (&out)[4]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) out[i] = atan_sqrt_deg(q[i] * ky2);
}
template <bool SQUARE> struct SlopeOpT {
    using in_t = float;
    using out_t = float;
    static constexpr int kOutputs = 1;
    using Params = SlopeParams;
    const Params &p;
    HornRow m2, m1;  // rows y-2, y-1 relative to the row being pushed
    __device__ explicit SlopeOpT(const Params &pp) : p(pp) {
#pragma unroll
        for (int i = 0; i < 4; ++i) m2.D[i] = m2.S[i] = m1.D[i] = m1.S[i] = 0.0;
    }
    __device__ __forceinline__ void step(const Row6<float> &row, Vec4<float> (&out)[1]) {
        const HornRow n = horn_row(row);
        float q[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            // dz_dx*8cs = (c+2f+i)-(a+2d+g) = D(y+1)+2D(y)+D(y-1);  dz_dy*8cs = S(y-1)-S(y+1)
            const double X = fma(2.0, m1.D[i], m2.D[i]) + n.D[i];
            const double Y = m2.S[i] - n.S[i];
            q[i] = slope_q<SQUARE>(X, Y, p);
        }
        slope_tail4(q, p.ky2, out[0].v);
        m2 = m1;
        m1 = n;
    }
};
using SlopeOp = SlopeOpT<false>;
using SlopeSqOp = SlopeOpT<true>;

// ------------------------------------------------------------------ aspect (aspect.py:56-90)
// X = 8*dz_dx, Y = 8*dz_dy, exact in f64; rounding them to f32 (6e-8) before the octant
// reduction is far inside the 1e-5 bar, and (float)X == 0 iff X == 0 for any raster whose
// cells are not denormal, so the flat (-1) mask is the reference's bit for bit.
__device__ __forceinline__ void aspect_tail4(const float (&u)[4], const float (&v)[4], float (&out)[4]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) out[i] = compass_deg(u[i], v[i]);
}
struct AspectOp {
    using in_t = float;
    using out_t = float;
    static constexpr int kOutputs = 1;
    struct Params {
        int unused;
    };
    HornRow m2, m1;
    __device__ explicit AspectOp(const Params &) {
#pragma unroll
        for (int i = 0; i < 4; ++i) m2.D[i] = m2.S[i] = m1.D[i] = m1.S[i] = 0.0;
    }
    __device__ __forceinline__ void step(const Row6<float> &row, Vec4<float> (&out)[1]) {
        const HornRow n = horn_row(row);
        float u[4], v[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const double X = fma(2.0, m1.D[i], m2.D[i]) + n.D[i];
            const double Y = n.S[i] - m2.S[i];  // a,b,c = row y-1 here (aspect.py:65-72)
            u[i] = (float)(-X);
            v[i] = (float)Y;
        }
        aspect_tail4(u, v, out[0].v);
        m2 = m1;
        m1 = n;
    }
};

// ------------------------------------------------------------------ curvature (curvature.py:31-41)
// The reference forms N+S and E+W in float32 (rounded) before promoting; reproduce that, then
// 4C - ns - ew is exact in f64 and only the final scale rounds.
struct CurvatureOp {
    using in_t = float;
    using out_t = float;
    static constexpr int kOutputs = 1;
    struct Params {
        double k;  // 100 / cellsize^2
        static Params make(double cellsize) {
            Params p;
            p.k = 100.0 / (cellsize * cellsize);
            return p;
        }
    };
    const Params &p;
    float n2[4];      // row y-2 centre cells
    Row6<float> r1;   // row y-1
    __device__ explicit CurvatureOp(const Params &pp) : p(pp) {
#pragma unroll
        for (int i = 0; i < 4; ++i) n2[i] = 0.f, r1.c[i] = 0.f;
        r1.l = r1.r = 0.f;
    }
    static __device__ __forceinline__ float eval(float ns, float ew, float c, double k) {
        // -2*(d+e) with d = ns/2 - c, e = ew/2 - c  ==  4c - ns - ew
        const double t = fma(4.0, (double)c, -(double)ns) - (double)ew;
        return (float)(t * k);
    }
    __device__ __forceinline__ void step(const Row6<float> &row, Vec4<float> (&out)[1]) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float ns = row.c[i] + n2[i];
            const float e = (i == 3) ? r1.r : r1.c[i + 1];
            const float w = (i == 0) ? r1.l : r1.c[i - 1];
            out[0].v[i] = eval(ns, e + w, r1.c[i], p.k);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) n2[i] = r1.c[i];
        r1 = row;
    }
};

// ------------------------------------------------------------------ hillshade (hillshade.py:20-35)
// With g = |grad|, slope = pi/2 - atan g and aspect = atan2(-gx, gy) the reference's
//   sin(alt) sin(slope) + cos(alt) cos(slope) cos((az - pi/2) - aspect)
// equals  [sin(alt) + cos(alt) (cosA gy - sinA gx)] / sqrt(1 + g^2),  A = az - pi/2,
// so no trigonometric function is needed per cell (all float32, like the reference's
// np.gradient / ufunc chain; agreement ~2e-7 absolute on values in [0, 1]).
struct HillshadeOp {
    using in_t = float;
    using out_t = float;
    static constexpr int kOutputs = 1;
    struct Params {
        float s0, cy, cx;  // sin(alt), 0.5*cos(alt)*cos(A), 0.5*cos(alt)*sin(A)
        static Params make(double azimuth, double angle_altitude) {
            // hillshade.py:23-27: azimuth = 360 - azimuth; rad conversions in Python float (f64)
            const double az = 360.0 - azimuth;
            const double azimuthrad = az * M_PI / 180.;
            const double altituderad = angle_altitude * M_PI / 180.;
            const double A = azimuthrad - M_PI / 2.;
            Params p;
            p.s0 = (float)sin(altituderad);
            p.cy = (float)(0.5 * cos(altituderad) * cos(A));
            p.cx = (float)(0.5 * cos(altituderad) * sin(A));
            return p;
        }
    };
    const Params &p;
    float n2[4];
    Row6<float> r1;
    __device__ explicit HillshadeOp(const Params &pp) : p(pp) {
#pragma unroll
        for (int i = 0; i < 4; ++i) n2[i] = 0.f, r1.c[i] = 0.f;
        r1.l = r1.r = 0.f;
    }
    static __device__ __forceinline__ float eval(float gx2, float gy2, const Params &p) {
        // gx2 = 2*d/drow, gy2 = 2*d/dcol
        const float q = fmaf(gx2, gx2, gy2 * gy2);
        const float rinv = rsqrt_approx(fmaf(0.25f, q, 1.0f));
        const float num = fmaf(p.cy, gy2, fmaf(-p.cx, gx2, p.s0));
        return fmaf(0.5f * num, rinv, 0.5f);
    }
    __device__ __forceinline__ void step(const Row6<float> &row, Vec4<float> (&out)[1]) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float e = (i == 3) ? r1.r : r1.c[i + 1];
            const float w = (i == 0) ? r1.l : r1.c[i - 1];
            out[0].v[i] = eval(row.c[i] - n2[i], e - w, p);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) n2[i] = r1.c[i];
        r1 = row;
    }
};

// ------------------------------------------------------------------ fused surface suite
// analytics.summarize_terrain (analytics.py:84-86): slope + aspect + curvature (+ hillshade)
// from ONE read of the DEM.  Output k is skipped when its pointer is NULL.
struct SuiteParams {
    SlopeParams slope;
    CurvatureOp::Params curv;
    HillshadeOp::Params hill;
};
template <bool SQUARE> struct SuiteOpT {
    using in_t = float;
    using out_t = float;
    static constexpr int kOutputs = 4;  // slope, aspect, curvature, hillshade
    using Params = SuiteParams;
    const Params &p;
    HornRow m2, m1;
    float n2[4];
    Row6<float> r1;
    __device__ explicit SuiteOpT(const Params &pp) : p(pp) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            m2.D[i] = m2.S[i] = m1.D[i] = m1.S[i] = 0.0;
            n2[i] = 0.f;
            r1.c[i] = 0.f;
        }
        r1.l = r1.r = 0.f;
    }
    __device__ __forceinline__ void step(const Row6<float> &row, Vec4<float> (&out)[4]) {
        const HornRow n = horn_row(row);
        float q[4], u[4], v[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const double X = fma(2.0, m1.D[i], m2.D[i]) + n.D[i];
            const double Ys = m2.S[i] - n.S[i];
            q[i] = slope_q<SQUARE>(X, Ys, p.slope);
            u[i] = (float)(-X);
            v[i] = (float)(-Ys);
            const float e = (i == 3) ? r1.r : r1.c[i + 1];
            const float w = (i == 0) ? r1.l : r1.c[i - 1];
            out[2].v[i] = CurvatureOp::eval(row.c[i] + n2[i], e + w, r1.c[i], p.curv.k);
            out[3].v[i] = HillshadeOp::eval(row.c[i] - n2[i], e - w, p.hill);
        }
        slope_tail4(q, p.slope.ky2, out[0].v);
        aspect_tail4(u, v, out[1].v);
        m2 = m1;
        m1 = n;
#pragma unroll
        for (int i = 0; i < 4; ++i) n2[i] = r1.c[i];
        r1 = row;
    }
};
using SuiteOp = SuiteOpT<false>;
using SuiteSqOp = SuiteOpT<true>;

// ------------------------------------------------------------------ 3x3 convolution (convolution.py:285-313)
// k = 3 runs on the warp-strip skeleton (HBM-bound) instead of the k x k tile kernel: float64
// accumulation in the reference's row-major tap order, NaN ring from the TMA fill.
struct Conv3Op {
    using in_t = float;
    using out_t = float;
    static constexpr int kOutputs = 1;
    struct Params {
        double w[9];
    };
    const Params &p;
    double r2[6], r1[6];  // rows y-2, y-1 widened to f64: left, 4 cells, right
    __device__ explicit Conv3Op(const Params &pp) : p(pp) {
#pragma unroll
        for (int i = 0; i < 6; ++i) r2[i] = r1[i] = 0.0;
    }
    __device__ __forceinline__ void step(const Row6<float> &row, Vec4<float> (&out)[1]) {
        double n[6];
        n[0] = (double)row.l;
#pragma unroll
        for (int i = 0; i < 4; ++i) n[i + 1] = (double)row.c[i];
        n[5] = (double)row.r;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            double acc = 0.0;
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) acc = fma(p.w[kx], r2[i + kx], acc);
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) acc = fma(p.w[3 + kx], r1[i + kx], acc);
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) acc = fma(p.w[6 + kx], n[i + kx], acc);
            out[0].v[i] = (float)acc;
        }
#pragma unroll
        for (int i = 0; i < 6; ++i) r2[i] = r1[i], r1[i] = n[i];
    }
};

// sum / cnt for cnt in 0..9 without a f64 division: multiply by a tabulated reciprocal and
// apply one FMA correction step (the quotient is then correctly rounded except in rare
// halfway cases; 0/0 gives NaN like np.divide).
// entry 0 is NaN: an empty window has s = 0 and 0 * NaN = NaN, like np.divide(0., 0)
__constant__ double kRcp9[10] = {
    __builtin_nan(""), 1.0, 1.0 / 2, 1.0 / 3, 1.0 / 4, 1.0 / 5, 1.0 / 6, 1.0 / 7, 1.0 / 8, 1.0 / 9};
__constant__ double kCnt9[10] = {0.0, 1.0, 2.0, 3.0, 4.0, 5.0, 6.0, 7.0, 8.0, 9.0};
// full window (9 valid cells): the same arithmetic with literal operands
template <typename TOUT> __device__ __forceinline__ TOUT div_full9(double s) {
    const double r9 = 1.0 / 9, q9 = s * r9;
    if constexpr (sizeof(TOUT) == 4) return (float)q9;
    else return fma(fma(-q9, 9.0, s), r9, q9);
}
template <typename TOUT> __device__ __forceinline__ TOUT div_count9(double s, int cnt) {
    const double r = kRcp9[cnt];
    const double q = s * r;
    if constexpr (sizeof(TOUT) == 4) {
        // float32 result: s * (1/n) is within one f64 ulp of s / n, so the f32 rounding agrees
        // with the oracle except when s / n sits within 1e-16 of an f32 rounding boundary
        return (float)q;
    } else {
        const double e = fma(-q, kCnt9[cnt], s);
        return fma(e, r, q);
    }
}

// ------------------------------------------------------------------ focal.mean (focal.py:44-67)
// 3x3 NaN-skipping mean over the window clamped to the raster (out-of-raster cells arrive
// as NaN and are skipped like any NaN); centre cells matching `excludes` are copied.
//
// Two paths per pushed row, chosen warp-uniformly (one vote):
//   * clean: no lane of the warp saw a NaN in this row nor in the two rows above -> every window
//     has 9 valid cells: unmasked f64 sums, one multiplication by 1/9, no counts, no selects;
//   * general: NaN -> 0 masking, per-cell counts, tabulated reciprocal, excludes.
// Both paths form the same sums in the same order, so which path a warp takes never changes a
// result (rasters without NaN just run ~2x fewer instructions: the kernel drops from issue-bound to
// HBM-bound).  Rows pushed on the clean path have count 3 per cell by definition; the count
// registers are only written on the general path and read through the row's clean flag.
template <typename T, typename TOUT = T, bool HAS_EX = false> struct FocalMeanOp {
    using in_t = T;
    using out_t = TOUT;
    static constexpr int kOutputs = 1;
    static constexpr int kMaxEx = 8;
    struct Params {
        double ex[kMaxEx];
        int n_ex;
        int ex_nan;  // some exclude is NaN
    };
    const Params &p;
    double s2[4], s1[4];  // horizontal 3-sums of rows y-2, y-1 (NaN -> 0)
    int c2[4], c1[4];     // matching counts (valid when the row's clean flag is false)
    bool clean2, clean1;  // warp-uniform: the row held no NaN for any lane of the warp
    T ctr[4];             // centre cells of row y-1
    __device__ explicit FocalMeanOp(const Params &pp) : p(pp), clean2(false), clean1(false) {
#pragma unroll
        for (int i = 0; i < 4; ++i) s2[i] = s1[i] = 0.0, c2[i] = c1[i] = 0, ctr[i] = (T)0;
    }
    __device__ __forceinline__ void step(const Row6<T> &row, Vec4<TOUT> (&out)[1]) {
        T w[6];
        w[0] = row.l; w[5] = row.r;
#pragma unroll
        for (int i = 0; i < 4; ++i) w[i + 1] = row.c[i];
        double g[6], hs[4];
#pragma unroll
        for (int i = 0; i < 6; ++i) g[i] = (double)w[i];
#pragma unroll
        for (int i = 0; i < 4; ++i) hs[i] = (g[i] + g[i + 1]) + g[i + 2];
        // a NaN anywhere in w[0..5] (or inf - inf) makes hs[0] + hs[3] NaN
        const double probe = hs[0] + hs[3];
        const bool row_clean = !HAS_EX && __all_sync(0xffffffffu, probe == probe);
        if (row_clean && clean1 && clean2) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const double sum = (s2[i] + s1[i]) + hs[i];
                out[0].v[i] = div_full9<TOUT>(sum);
                s2[i] = s1[i]; s1[i] = hs[i];
            }
        } else {
            double f[6];
            int m[6];
#pragma unroll
            for (int i = 0; i < 6; ++i) {
                const bool ok = (w[i] == w[i]);
                f[i] = ok ? g[i] : 0.0;
                m[i] = ok ? 1 : 0;
            }
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const double hsm = (f[i] + f[i + 1]) + f[i + 2];
                const int hc = m[i] + m[i + 1] + m[i + 2];
                const double sum = (s2[i] + s1[i]) + hsm;
                const int cnt = (clean2 ? 3 : c2[i]) + (clean1 ? 3 : c1[i]) + hc;
                const T c = ctr[i];
                bool excl;
                if constexpr (HAS_EX) {  // arbitrary exclude lists: rare, kept off the default path
                    excl = (p.ex_nan != 0) && !(c == c);
                    for (int k = 0; k < p.n_ex; ++k) excl = excl || ((double)c == p.ex[k]);
                } else {  // the default excludes=[nan]
                    excl = !(c == c);
                }
                const TOUT mean = div_count9<TOUT>(sum, cnt);
                out[0].v[i] = excl ? (TOUT)c : mean;
                s2[i] = s1[i]; s1[i] = hsm;
                c2[i] = clean1 ? 3 : c1[i]; c1[i] = hc;
            }
        }
        clean2 = clean1;
        clean1 = row_clean;
#pragma unroll
        for (int i = 0; i < 4; ++i) ctr[i] = row.c[i];
    }
};

}  // namespace xrs

// surface_ops.cuh -- per-row operators for the 3x3 skeleton (stencil3.cuh).
//
// Numerics follow the reference's *CPU* kernels, which do the Horn sums in float64 because
// Numba promotes `2 * f32` (SURVEY.md section 0 fact 5): the column differences / weighted row
// sums are formed in f64 (sums of <= 8 float32 values: exact whenever the window's cells lie
// within a factor 2^26 of each other), so re-associating them row by row changes nothing there.
// Where a window mixes terrain with a fill beyond that range (a row of -FLT_MAX), the reference's
// column-by-column X rounds the terrain away and these row differences do not: a documented
// deviation (DESIGN.md 4.1, "Fill values"); the transcendental
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
// X = 8*dz_dx, Y = 8*dz_dy in f64; rounding them to f32 (6e-8) before the octant reduction is
// far inside the 1e-5 bar, and (float)X == 0 iff X == 0 (X is 0 or at least 2^-149, which f32
// keeps) for any raster whose cells are not denormal, so the flat (-1) mask is the reference's bit
// for bit.  Denormal cells are not served: compass_pre's ftz reciprocal flushes a denormal sum.
//
// compass_uv4 gives compass_deg its (u, v) = (-X, Y) in f32.  Only their ratio and signs matter.
// Next to a fill value such as -FLT_MAX the larger sum exceeds 2^125, where compass_pre's
// reciprocal would flush to zero, or FLT_MAX, where the conversion would give inf; such a pair is
// scaled by 2^-8 in f64 first (exact, and the flat test cannot change: the pair is far from 0).
// An infinite sum (next to an infinite cell) counts as +-1 and a finite one as +-0, which is what
// the reference's float64 atan2 gives for them.
// compass_uv4 rounds the four cells of a lane and returns the largest |u|, |v| (7 FMNMX); only when
// it exceeds 2^125 (one compare and one branch per lane) does compass_wide4 rewrite the wide pairs,
// out of line so that the hot loop keeps its registers.
__device__ __noinline__ float2 compass_uv_wide(double X, double Y, float u, float v) {
    if (!(fmaxf(fabsf(u), fabsf(v)) > 0x1p125f)) return make_float2(u, v);   // fmaxf drops a NaN: it propagates
    const bool ix = isinf(X), iy = isinf(Y);
    if (ix || iy)
        return make_float2(ix ? copysignf(1.0f, u) : (float)(X * -0.0),   // X * 0 keeps a NaN
                           iy ? copysignf(1.0f, v) : (float)(Y * 0.0));
    return make_float2((float)(X * -0x1p-8), (float)(Y * 0x1p-8));
}
__device__ __forceinline__ float compass_uv4(const double (&X)[4], const double (&Y)[4], float (&u)[4],
                                             float (&v)[4]) {
    float m = 0.0f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        u[i] = (float)(-X[i]);
        v[i] = (float)Y[i];
        m = fmaxf(m, fmaxf(fabsf(u[i]), fabsf(v[i])));
    }
    return m;
}
constexpr float kCompassWide = 0x1p125f;
__device__ __forceinline__ void compass_wide4(const double (&X)[4], const double (&Y)[4], float (&u)[4],
                                              float (&v)[4]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float2 w = compass_uv_wide(X[i], Y[i], u[i], v[i]);
        u[i] = w.x;
        v[i] = w.y;
    }
}
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
        double X[4], Y[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            X[i] = fma(2.0, m1.D[i], m2.D[i]) + n.D[i];
            Y[i] = n.S[i] - m2.S[i];  // a,b,c = row y-1 here (aspect.py:65-72)
        }
        if (compass_uv4(X, Y, u, v) > kCompassWide) compass_wide4(X, Y, u, v);   // rare: next to fills
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
    // Where q = gx2^2 + gy2^2 overflows f32 (a fill value such as -FLT_MAX next to terrain, |grad| > 9e18) the
    // closed form would give 0.5 or NaN.  Its limit for a large gradient, 0.5 + (cy gy2 - cx gx2) / |(gx2, gy2)|,
    // is the reference's value there: its f32 x*x + y*y overflows as well (slope 0) and cos(A - aspect) is the
    // same direction cosine.  Only the direction matters, so the pair is scaled by 2^-100 (it is then below
    // 2^28, above 2^-38); an infinite component (an infinite cell) counts as +-1 against 0, as in atan2.
    static __device__ __noinline__ float steep(float gx2, float gy2, const Params &p) {
        const bool ix = isinf(gx2), iy = isinf(gy2);
        const float s = (ix || iy) ? 0.0f : 0x1p-100f;
        const float x = ix ? copysignf(1.0f, gx2) : gx2 * s;
        const float y = iy ? copysignf(1.0f, gy2) : gy2 * s;
        return fmaf(fmaf(p.cy, y, -p.cx * x), rsqrt_approx(fmaf(x, x, y * y)), 0.5f);
    }
    // the four cells of a lane (gx2 = 2*d/drow, gy2 = 2*d/dcol, q their squared norm); returns the largest q,
    // which is inf where steep4 has to rewrite a cell (3 FMNMX)
    static __device__ __forceinline__ float eval4(const float (&gx2)[4], const float (&gy2)[4], const Params &p,
                                                  float (&q)[4], float (&out)[4]) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            q[i] = fmaf(gx2[i], gx2[i], gy2[i] * gy2[i]);
            const float rinv = rsqrt_approx(fmaf(0.25f, q[i], 1.0f));
            const float num = fmaf(p.cy, gy2[i], fmaf(-p.cx, gx2[i], p.s0));
            out[i] = fmaf(0.5f * num, rinv, 0.5f);
        }
        return fmaxf(fmaxf(q[0], q[1]), fmaxf(q[2], q[3]));
    }
    static __device__ __forceinline__ void steep4(const float (&gx2)[4], const float (&gy2)[4], const Params &p,
                                                  const float (&q)[4], float (&out)[4]) {
#pragma unroll
        for (int i = 0; i < 4; ++i)
            if (q[i] == INFINITY) out[i] = steep(gx2[i], gy2[i], p);
    }
    __device__ __forceinline__ void step(const Row6<float> &row, Vec4<float> (&out)[1]) {
        float gx2[4], gy2[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float e = (i == 3) ? r1.r : r1.c[i + 1];
            const float w = (i == 0) ? r1.l : r1.c[i - 1];
            gx2[i] = row.c[i] - n2[i];
            gy2[i] = e - w;
        }
        float q[4];
        if (eval4(gx2, gy2, p, q, out[0].v) == INFINITY) steep4(gx2, gy2, p, q, out[0].v);   // rare: next to fills
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
        float q[4], u[4], v[4], gx2[4], gy2[4];
        double X[4], Y[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            X[i] = fma(2.0, m1.D[i], m2.D[i]) + n.D[i];
            const double Ys = m2.S[i] - n.S[i];
            q[i] = slope_q<SQUARE>(X[i], Ys, p.slope);
            Y[i] = -Ys;
            const float e = (i == 3) ? r1.r : r1.c[i + 1];
            const float w = (i == 0) ? r1.l : r1.c[i - 1];
            out[2].v[i] = CurvatureOp::eval(row.c[i] + n2[i], e + w, r1.c[i], p.curv.k);
            gx2[i] = row.c[i] - n2[i];
            gy2[i] = e - w;
        }
        float qh[4];
        const float m = compass_uv4(X, Y, u, v);
        const float qmax = HillshadeOp::eval4(gx2, gy2, p.hill, qh, out[3].v);
        if (m > kCompassWide || qmax == INFINITY) {   // rare: next to fills; one test for aspect and hillshade
            compass_wide4(X, Y, u, v);
            HillshadeOp::steep4(gx2, gy2, p.hill, qh, out[3].v);
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
// A window of -0.0 cells sums to -0.0 here but to +0.0 in the reference, whose sum starts at +0.0:
// the float32 quotient is fma(s, r, +0.0), the same bits as s * r except that -0.0 becomes +0.0 (the
// float64 correction step below does the same).  An infinite sum (infinite cells, or float64 cells
// beyond DBL_MAX / 9 in total) skips the correction step, whose residual would be inf - inf = NaN.
// full window (9 valid cells): the same arithmetic with literal operands
template <typename TOUT> __device__ __forceinline__ TOUT div_full9(double s) {
    const double r9 = 1.0 / 9;
    if constexpr (sizeof(TOUT) == 4) {
        return (float)fma(s, r9, 0.0);
    } else {
        const double q9 = s * r9, e = fma(-q9, 9.0, s);
        return e == e ? fma(e, r9, q9) : q9;
    }
}
template <typename TOUT> __device__ __forceinline__ TOUT div_count9(double s, int cnt) {
    const double r = kRcp9[cnt];
    if constexpr (sizeof(TOUT) == 4) {
        // float32 result: s * (1/n) is within one f64 ulp of s / n, so the f32 rounding agrees
        // with the oracle except when s / n sits within 1e-16 of an f32 rounding boundary
        return (float)fma(s, r, 0.0);
    } else {
        const double q = s * r, e = fma(-q, kCnt9[cnt], s);
        return e == e ? fma(e, r, q) : q;
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

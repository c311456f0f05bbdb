/*
 * xrs_oracle.c -- CPU restatement of the xarray-spatial dense-stencil hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under xarray-spatial_b200/ (the product) may
 * import, link or call this file.  It is used by tests/ (as the checker), by
 * __graft_entry__.smoke() and by bench.py's cpu_baseline / --impl reference legs.
 *
 * Every function restates, in plain C, the arithmetic the reference's Numba-CPU
 * (or NumPy) path performs, INCLUDING the float64 promotions Numba applies to
 * "float32" kernels (SURVEY.md section 0 fact 5).  Citations are file:line in
 * the reference's xrspatial/.  Parity is PINNED: tests/test_oracle_golden.py checks
 * this file against (a) the literal QGIS / hand-derived arrays of the reference's own
 * test-suite and docstrings and (b) the .npz files under tests/golden/, which were produced by running
 * the unmodified reference kernels in this container (oracle/make_golden.py).
 *
 * Threading: every entry point takes `nthreads`.  1 reproduces the stock reference
 * (ngjit has no parallel=True, utils.py:31); >1 splits output rows over OpenMP
 * threads, which is what dask.map_overlap would do with the same nogil kernels
 * (slope.py:86-98).  Results do not depend on nthreads (each cell is independent).
 *
 * Build: see oracle/Makefile  (gcc -O2 -fopenmp -fno-fast-math -ffp-contract=off).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define XO_EXPORT __attribute__((visibility("default")))

static void fill_nan_f32(float *p, int64_t n) {
    for (int64_t i = 0; i < n; ++i) p[i] = NAN;
}

/* ------------------------------------------------------------------ slope
 * slope.py:56-76 `_cpu`.  a,b,c = row y+1; g,h,i = row y-1.  `2 * f` with an int
 * literal promotes the float32 element to float64, so the whole expression is f64;
 * np.arctan(f64) * 57.29578 is f64 and is rounded to f32 on store.  `** .5` is
 * pow(x, .5); sqrt() agrees with it to the last bit except on a measure-zero set
 * (validated against the reference in tests).
 */
XO_EXPORT void xo_slope_f32(const float *in, float *out, int64_t H, int64_t W,
                            double csx, double csy, int nthreads) {
    fill_nan_f32(out, H * W);
#pragma omp parallel for num_threads(nthreads) schedule(static)
    for (int64_t y = 1; y < H - 1; ++y) {
        const float *up = in + (y + 1) * W, *mid = in + y * W, *dn = in + (y - 1) * W;
        for (int64_t x = 1; x < W - 1; ++x) {
            double a = up[x - 1], b = up[x], c = up[x + 1];
            double d = mid[x - 1], f = mid[x + 1];
            double g = dn[x - 1], h = dn[x], i = dn[x + 1];
            double dz_dx = ((c + 2 * f + i) - (a + 2 * d + g)) / (8 * csx);
            double dz_dy = ((g + 2 * h + i) - (a + 2 * b + c)) / (8 * csy);
            double p = sqrt(dz_dx * dz_dx + dz_dy * dz_dy);
            out[y * W + x] = (float)(atan(p) * 57.29578);
        }
    }
}

/* ------------------------------------------------------------------ aspect
 * aspect.py:56-90 `_run_numpy`.  a,b,c = row y-1; g,h,i = row y+1; /8 (no cellsize);
 * flat -> -1; atan2(dz_dy, -dz_dx) * (180/pi) (RADIAN, aspect.py:49), compass fold.
 * The CPU path has no 359.999 clamp (that is GPU-only, aspect.py:121) -- follow CPU.
 */
XO_EXPORT void xo_aspect_f32(const float *in, float *out, int64_t H, int64_t W, int nthreads) {
    const double RADIAN = 180.0 / M_PI;
    fill_nan_f32(out, H * W);
#pragma omp parallel for num_threads(nthreads) schedule(static)
    for (int64_t y = 1; y < H - 1; ++y) {
        const float *up = in + (y - 1) * W, *mid = in + y * W, *dn = in + (y + 1) * W;
        for (int64_t x = 1; x < W - 1; ++x) {
            double a = up[x - 1], b = up[x], c = up[x + 1];
            double d = mid[x - 1], f = mid[x + 1];
            double g = dn[x - 1], h = dn[x], i = dn[x + 1];
            double dz_dx = ((c + 2 * f + i) - (a + 2 * d + g)) / 8;
            double dz_dy = ((g + 2 * h + i) - (a + 2 * b + c)) / 8;
            float r;
            if (dz_dx == 0 && dz_dy == 0) {
                r = -1.f;
            } else {
                double asp = atan2(dz_dy, -dz_dx) * RADIAN;
                if (asp < 0) r = (float)(90.0 - asp);
                else if (asp > 90.0) r = (float)(360.0 - asp + 90.0);
                else r = (float)(90.0 - asp);
            }
            out[y * W + x] = r;
        }
    }
}

/* --------------------------------------------------------------- curvature
 * curvature.py:31-41 `_cpu` (input already float32, :47).  The neighbour sums
 * `data[y+1,x] + data[y-1,x]` are float32 + float32 = float32 (ROUNDED in f32); only
 * the `/ 2` promotes to f64 (checked bit-for-bit against the reference: computing the
 * sums in f64 differs from it by up to 1e-3 relative).
 */
XO_EXPORT void xo_curvature_f32(const float *in, float *out, int64_t H, int64_t W,
                                double cellsize, int nthreads) {
    fill_nan_f32(out, H * W);
#pragma omp parallel for num_threads(nthreads) schedule(static)
    for (int64_t y = 1; y < H - 1; ++y) {
        for (int64_t x = 1; x < W - 1; ++x) {
            double ctr = in[y * W + x];
            float ns = in[(y + 1) * W + x] + in[(y - 1) * W + x];
            float ew = in[y * W + x + 1] + in[y * W + x - 1];
            double d = (double)ns / 2 - ctr;
            double e = (double)ew / 2 - ctr;
            out[y * W + x] = (float)(-2 * (d + e) * 100 / (cellsize * cellsize));
        }
    }
}

/* --------------------------------------------------------------- hillshade
 * hillshade.py:20-35 `_run_numpy` (pure NumPy).  np.gradient on float32 (central
 * differences /2, cellsize ignored); sqrt/arctan/arctan2/sin/cos of float32 arrays
 * stay float32; np.sin(py_float) / np.cos(py_float) are np.float64 scalars, so the
 * final combine and the result are float64 under NumPy 2 (SURVEY.md 8a row a5).
 * NumPy may use SIMD (SVML) float32 transcendentals that differ from libm by a few
 * f32 ulp; the oracle therefore matches the reference to ~1e-6 abs, not bit-for-bit.
 * Border rows/cols are NaN (:33-34) so the one-sided edge gradients never matter.
 */
XO_EXPORT void xo_hillshade_f32(const float *in, double *out, int64_t H, int64_t W,
                                double azimuth, double angle_altitude, int nthreads) {
    const double az = 360.0 - azimuth;
    const double azimuthrad = az * M_PI / 180.;
    const double altituderad = angle_altitude * M_PI / 180.;
    const double sin_alt = sin(altituderad), cos_alt = cos(altituderad);
    const float half_pi_f = (float)(M_PI / 2.);
    const float az_m = (float)(azimuthrad - M_PI / 2.); /* weak python float -> f32 */
    for (int64_t i = 0; i < H * W; ++i) out[i] = NAN;
#pragma omp parallel for num_threads(nthreads) schedule(static)
    for (int64_t y = 1; y < H - 1; ++y) {
        for (int64_t x = 1; x < W - 1; ++x) {
            float gx = (in[(y + 1) * W + x] - in[(y - 1) * W + x]) / 2.0f; /* d/d-row */
            float gy = (in[y * W + x + 1] - in[y * W + x - 1]) / 2.0f;     /* d/d-col */
            float slope = half_pi_f - atanf(sqrtf(gx * gx + gy * gy));
            float aspect = atan2f(-gx, gy);
            double shaded = sin_alt * (double)sinf(slope) +
                            cos_alt * (double)cosf(slope) * (double)cosf(az_m - aspect);
            out[y * W + x] = (shaded + 1) / 2;
        }
    }
}

/* -------------------------------------------------------------- convolve_2d
 * convolution.py:285-313 `_convolve_2d_numpy`: correlation, f64 accumulator starting
 * at 0.0, row-major order over the window, product kernel(f64) * data(f32->f64);
 * a NaN ring of (kh//2, kw//2); NaN inputs propagate.
 */
XO_EXPORT void xo_convolve2d_f32(const float *in, const double *kernel, int kh, int kw,
                                 float *out, int64_t H, int64_t W, int nthreads) {
    const int ry = kh / 2, rx = kw / 2;
    fill_nan_f32(out, H * W);
#pragma omp parallel for num_threads(nthreads) schedule(static)
    for (int64_t i = ry; i < H - ry; ++i) {
        for (int64_t j = rx; j < W - rx; ++j) {
            double num = 0.0;
            for (int ii = 0; ii < kh; ++ii)
                for (int jj = 0; jj < kw; ++jj)
                    num += kernel[ii * kw + jj] * (double)in[(i + ii - ry) * W + (j + jj - rx)];
            out[i * W + j] = (float)num;
        }
    }
}

/* The project's CUDA convolve kernels restated: the same row-major tap order and +0.0 start, but every
 * step is one fused multiply-add, acc = fma(w, (double)x, acc), and out-of-raster taps are NaN (so the
 * border ring is NaN whatever the weights).  The GPU kernels must equal this bit for bit; it differs from
 * xo_convolve2d_f32 (two roundings per tap) by float64 rounding only. */
XO_EXPORT void xo_convolve2d_fma_f32(const float *in, const double *kernel, int kh, int kw,
                                     float *out, int64_t H, int64_t W, int nthreads) {
    const int ry = kh / 2, rx = kw / 2;
#pragma omp parallel for num_threads(nthreads) schedule(static)
    for (int64_t i = 0; i < H; ++i) {
        for (int64_t j = 0; j < W; ++j) {
            double acc = 0.0;
            for (int ii = 0; ii < kh; ++ii)
                for (int jj = 0; jj < kw; ++jj) {
                    const int64_t y = i + ii - ry, x = j + jj - rx;
                    const double v = (y >= 0 && y < H && x >= 0 && x < W) ? (double)in[y * W + x] : (double)NAN;
                    acc = fma(kernel[ii * kw + jj], v, acc);
                }
            out[i * W + j] = (float)acc;
        }
    }
}

/* --------------------------------------------------------------- focal.mean
 * focal.py:44-67 `_mean_numpy` (one pass; focal.py:257-259 casts to float64 first and
 * loops passes).  Centre in `excludes` (NaN-aware equality, :37-41) -> copy; else
 * np.nanmean (f64 accumulator, row-major, divide by count; 0/0 -> NaN) of the 3x3
 * window clamped to the raster.
 */
XO_EXPORT void xo_focal_mean_f64(const double *in, double *out, int64_t H, int64_t W,
                                 const double *excludes, int n_ex, int nthreads) {
#pragma omp parallel for num_threads(nthreads) schedule(static)
    for (int64_t y = 0; y < H; ++y) {
        for (int64_t x = 0; x < W; ++x) {
            double v = in[y * W + x];
            int ex = 0;
            for (int k = 0; k < n_ex; ++k)
                if (v == excludes[k] || (isnan(v) && isnan(excludes[k]))) { ex = 1; break; }
            if (ex) { out[y * W + x] = v; continue; }
            int64_t l = x - 1 < 0 ? 0 : x - 1, r = x + 2 > W ? W : x + 2;
            int64_t b = y - 1 < 0 ? 0 : y - 1, t = y + 2 > H ? H : y + 2;
            double c = 0.0; int64_t cnt = 0;
            for (int64_t yy = b; yy < t; ++yy)
                for (int64_t xx = l; xx < r; ++xx) {
                    double u = in[yy * W + xx];
                    if (!isnan(u)) { c += u; cnt++; }
                }
            out[y * W + x] = c / (double)cnt; /* np.divide: 0/0 = nan */
        }
    }
}

/* ---------------------------------------------------- focal.apply / focal_stats
 * focal.py:305-326 `_apply_numpy` with the built-in reducers :268-302.  Input cast to
 * f32; for every cell a kh x kw scratch is NaN-filled and receives data where the
 * kernel value == 1 and the position is in bounds; the reducer sees the scratch in
 * row-major order.  Numba semantics (numba/np/arraymath.py): nanmean / nanvar use an
 * f64 accumulator (nanvar two-pass around the f64 mean, nanstd = nanvar**.5), nansum
 * accumulates in the array dtype (f32), nanmin/nanmax skip NaN (all-NaN -> NaN),
 * range = nanmax - nanmin in f32.  The result is stored to an f32 output.
 */
enum { XO_STAT_MEAN = 0, XO_STAT_SUM = 1, XO_STAT_MIN = 2, XO_STAT_MAX = 3,
       XO_STAT_STD = 4, XO_STAT_RANGE = 5, XO_STAT_VAR = 6 };

XO_EXPORT void xo_focal_apply_f32(const float *in, const double *kernel, int kh, int kw,
                                  int stat, float *out, int64_t H, int64_t W, int nthreads) {
    const int hr = kh / 2, hc = kw / 2;
#pragma omp parallel for num_threads(nthreads) schedule(static)
    for (int64_t y = 0; y < H; ++y) {
        float *scratch = (float *)malloc(sizeof(float) * kh * kw);
        for (int64_t x = 0; x < W; ++x) {
            for (int k = 0; k < kh * kw; ++k) scratch[k] = NAN;
            for (int ky = 0; ky < kh; ++ky)
                for (int kx = 0; kx < kw; ++kx) {
                    int64_t yy = y - hr + ky, xx = x - hc + kx;
                    if (yy >= 0 && yy < H && xx >= 0 && xx < W && kernel[ky * kw + kx] == 1)
                        scratch[ky * kw + kx] = in[yy * W + xx];
                }
            const int n = kh * kw;
            float res;
            if (stat == XO_STAT_MEAN || stat == XO_STAT_VAR || stat == XO_STAT_STD) {
                double c = 0.0; int64_t cnt = 0;
                for (int k = 0; k < n; ++k) if (!isnan(scratch[k])) { c += scratch[k]; cnt++; }
                double m = c / (double)cnt;
                if (stat == XO_STAT_MEAN) res = (float)m;
                else {
                    double ssd = 0.0; int64_t c2 = 0;
                    for (int k = 0; k < n; ++k) if (!isnan(scratch[k])) {
                        double val = (double)scratch[k] - m; ssd += val * val; c2++; }
                    double var = ssd / (double)c2;
                    res = (float)(stat == XO_STAT_VAR ? var : sqrt(var));
                }
            } else if (stat == XO_STAT_SUM) {
                float c = 0.f;
                for (int k = 0; k < n; ++k) if (!isnan(scratch[k])) c += scratch[k];
                res = c;
            } else {
                float mn = scratch[0], mx = scratch[0];
                for (int k = 1; k < n; ++k) {
                    float v = scratch[k];
                    if (!isnan(v)) { if (!(mn < v)) mn = v; if (!(mx > v)) mx = v; }
                }
                res = stat == XO_STAT_MIN ? mn : stat == XO_STAT_MAX ? mx : mx - mn;
            }
            out[y * W + x] = res;
        }
        free(scratch);
    }
}

/* ------------------------------------------------------------ multispectral
 * All inputs are float32 (callers .astype('f4'), e.g. multispectral.py:727); outputs are
 * float32 pre-filled with NaN and left NaN where the denominator is 0.
 */
/* multispectral.py:825-841 `_normalized_ratio_cpu` (ndvi, nbr, nbr2, ndmi): pure f32. */
XO_EXPORT void xo_normalized_ratio_f32(const float *a, const float *b, float *out, int64_t n,
                                       int nthreads) {
#pragma omp parallel for num_threads(nthreads) schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        float num = a[i] - b[i], den = a[i] + b[i];
        out[i] = (den == 0.0f) ? NAN : num / den;
    }
}
/* multispectral.py:876-890 `_savi_cpu` with a Python float soil_factor: numerator f32,
 * nir + red (f32) + soil_factor and the rest of the denominator f64.  Numba sums
 * nir + red + soil_factor in f32 instead when soil_factor is a float32, int8, int16, uint8 or
 * bool; the device kernel follows that (its f32_sum flag), this oracle only the float64 sum. */
XO_EXPORT void xo_savi_f32(const float *nir, const float *red, double soil, float *out,
                           int64_t n, int nthreads) {
#pragma omp parallel for num_threads(nthreads) schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        float num = nir[i] - red[i];
        double soma = (double)(nir[i] + red[i]) + soil;
        double den = soma * (1.0 + soil);
        out[i] = (den != 0.0) ? (float)((double)num / den) : NAN;
    }
}
/* multispectral.py:175-188 `_evi_cpu`: c1,c2,L,G Python floats (or ints) -> f64 terms. */
XO_EXPORT void xo_evi_f32(const float *nir, const float *red, const float *blue, double c1,
                          double c2, double soil, double gain, float *out, int64_t n,
                          int nthreads) {
#pragma omp parallel for num_threads(nthreads) schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        float num = nir[i] - red[i];
        double den = (double)nir[i] + c1 * (double)red[i] - c2 * (double)blue[i] + soil;
        out[i] = (den != 0.0) ? (float)(gain * ((double)num / den)) : NAN;
    }
}
/* multispectral.py:29-43 `_arvi_cpu`: 2.0 * red is f64. */
XO_EXPORT void xo_arvi_f32(const float *nir, const float *red, const float *blue, float *out,
                           int64_t n, int nthreads) {
#pragma omp parallel for num_threads(nthreads) schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        double num = ((double)nir[i] - (2.0 * (double)red[i])) + (double)blue[i];
        double den = ((double)nir[i] + (2.0 * (double)red[i])) + (double)blue[i];
        out[i] = (den != 0.0) ? (float)(num / den) : NAN;
    }
}
/* multispectral.py:350-360 `_gci_cpu`: nir / green is f32, `- 1` (int) promotes to f64. */
XO_EXPORT void xo_gci_f32(const float *nir, const float *green, float *out, int64_t n,
                          int nthreads) {
#pragma omp parallel for num_threads(nthreads) schedule(static)
    for (int64_t i = 0; i < n; ++i)
        out[i] = (green[i] != 0) ? (float)((double)(nir[i] / green[i]) - 1) : NAN;
}
/* multispectral.py:1017-1030 `_sipi_cpu`: pure f32. */
XO_EXPORT void xo_sipi_f32(const float *nir, const float *red, const float *blue, float *out,
                           int64_t n, int nthreads) {
#pragma omp parallel for num_threads(nthreads) schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        float num = nir[i] - blue[i], den = nir[i] - red[i];
        out[i] = (den != 0.0f) ? num / den : NAN;
    }
}
/* multispectral.py:1160-1173 `_ebbi_cpu`: np.sqrt(f32) stays f32, 10 * (int) -> f64. */
XO_EXPORT void xo_ebbi_f32(const float *red, const float *swir, const float *tir, float *out,
                           int64_t n, int nthreads) {
#pragma omp parallel for num_threads(nthreads) schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        float num = swir[i] - red[i];
        double den = 10 * (double)sqrtf(swir[i] + tir[i]);
        out[i] = (den != 0.0) ? (float)((double)num / den) : NAN;
    }
}

/* ------------------------------------------------- geodesic slope / aspect
 * geodesic.py:40-231: every 3x3 neighbourhood is converted from (lat, lon, elevation) to ECEF
 * (:40-52), projected into the local East/North/Up frame of the centre cell, corrected for the
 * Earth's curvature (u += (e^2 + n^2) / (2 R_mean)) and fitted with u = A e + B n (+ C) by
 * centred least squares (:55-131); slope = atan(sqrt(A^2 + B^2)) in degrees (:134-145), aspect =
 * atan2(-A, -B) folded to [0, 360), -1 when sqrt(A^2 + B^2) < 1e-7 (:148-172).  All float64;
 * a NaN anywhere in the 3x3 elevations gives NaN; 1-cell NaN ring; float32 output.
 * elev / lat / lon are (H, W) float64 arrays (the `stacked` channels of :179-231). */
static void geo_ecef(double lat_rad, double lon_rad, double h, double a2, double b2, double *X, double *Y,
                     double *Z) {
    const double cos_lat = cos(lat_rad), sin_lat = sin(lat_rad), cos_lon = cos(lon_rad), sin_lon = sin(lon_rad);
    const double N = a2 / sqrt(a2 * cos_lat * cos_lat + b2 * sin_lat * sin_lat);
    *X = (N + h) * cos_lat * cos_lon;
    *Y = (N + h) * cos_lat * sin_lon;
    *Z = (b2 / a2 * N + h) * sin_lat;
}

static int geo_fit(const double *elev, const double *lat, const double *lon, int64_t W, int64_t y, int64_t x,
                   double a2, double b2, double z_factor, double inv_2r, double *A, double *B) {
    const double deg2rad = 3.141592653589793 / 180.0;
    double ne[9], nl[9], no[9];
    int idx = 0;
    for (int dy = -1; dy <= 1; ++dy)
        for (int dx = -1; dx <= 1; ++dx) {
            ne[idx] = elev[(y + dy) * W + x + dx];
            nl[idx] = lat[(y + dy) * W + x + dx];
            no[idx] = lon[(y + dy) * W + x + dx];
            idx++;
        }
    for (int k = 0; k < 9; ++k)
        if (ne[k] != ne[k]) return 0;
    const double lat_c = lat[y * W + x] * deg2rad, lon_c = lon[y * W + x] * deg2rad;
    double Xc, Yc, Zc;
    geo_ecef(lat_c, lon_c, elev[y * W + x] * z_factor, a2, b2, &Xc, &Yc, &Zc);
    const double cos_lat = cos(lat_c), sin_lat = sin(lat_c), cos_lon = cos(lon_c), sin_lon = sin(lon_c);
    const double ex = -sin_lon, ey = cos_lon, ez = 0.0;
    const double nx = -sin_lat * cos_lon, ny = -sin_lat * sin_lon, nz = cos_lat;
    const double ux = cos_lat * cos_lon, uy = cos_lat * sin_lon, uz = sin_lat;
    double e9[9], n9[9], u9[9];
    for (int k = 0; k < 9; ++k) {
        double Xk, Yk, Zk;
        geo_ecef(nl[k] * deg2rad, no[k] * deg2rad, ne[k] * z_factor, a2, b2, &Xk, &Yk, &Zk);
        const double dx = Xk - Xc, dy = Yk - Yc, dz = Zk - Zc;
        const double ek = dx * ex + dy * ey + dz * ez;
        const double nk = dx * nx + dy * ny + dz * nz;
        double uk = dx * ux + dy * uy + dz * uz;
        uk += (ek * ek + nk * nk) * inv_2r;
        e9[k] = ek; n9[k] = nk; u9[k] = uk;
    }
    double me = 0.0, mn = 0.0, mu = 0.0;
    for (int k = 0; k < 9; ++k) { me += e9[k]; mn += n9[k]; mu += u9[k]; }
    const double inv9 = 1.0 / 9.0;
    me *= inv9; mn *= inv9; mu *= inv9;
    double See = 0.0, Snn = 0.0, Sen = 0.0, Seu = 0.0, Snu = 0.0;
    for (int k = 0; k < 9; ++k) {
        const double de = e9[k] - me, dn = n9[k] - mn, du = u9[k] - mu;
        See += de * de; Snn += dn * dn; Sen += de * dn; Seu += de * du; Snu += dn * du;
    }
    const double det = See * Snn - Sen * Sen;
    if (fabs(det) < 1e-30) { *A = 0.0; *B = 0.0; return 1; }
    *A = (Seu * Snn - Snu * Sen) / det;
    *B = (Snu * See - Seu * Sen) / det;
    return 1;
}

XO_EXPORT void xo_geodesic_f64(const double *elev, const double *lat, const double *lon, float *out, int64_t H,
                               int64_t W, double z_factor, int want_aspect, int nthreads) {
    const double a2 = 6378137.0 * 6378137.0, b2 = 6356752.314245 * 6356752.314245;
    const double inv_2r = 1.0 / (2.0 * 6370994.884953014);
    fill_nan_f32(out, H * W);
#pragma omp parallel for num_threads(nthreads) schedule(static)
    for (int64_t y = 1; y < H - 1; ++y)
        for (int64_t x = 1; x < W - 1; ++x) {
            double A, B;
            if (!geo_fit(elev, lat, lon, W, y, x, a2, b2, z_factor, inv_2r, &A, &B)) continue;  /* NaN */
            if (!want_aspect) {
                out[y * W + x] = (float)(atan(sqrt(A * A + B * B)) * (180.0 / 3.141592653589793));
            } else {
                if (sqrt(A * A + B * B) < 1e-7) { out[y * W + x] = -1.0f; continue; }
                double deg = atan2(-A, -B) * (180.0 / 3.141592653589793);
                if (deg < 0) deg += 360.0;
                if (deg >= 360.0) deg -= 360.0;
                out[y * W + x] = (float)deg;
            }
        }
}

XO_EXPORT int xo_max_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

/* ------------------------------------------------------------------ benchmark DEM
 * Not reference arithmetic: the host twin of the product's benchmark-input generator
 * (xarray-spatial_b200/csrc/synth.cu -- 12 octaves of smoothstep-interpolated lattice value
 * noise, a pure function of (seed, global row, global col)), so that bench.py's CPU arms can
 * produce the SAME DEM window without touching the CUDA library.  Agrees with the device
 * generator to float32 rounding (exp2f / FMA-free float arithmetic), checked in the GPU tests.
 */
static uint32_t xo_hash3(uint32_t x, uint32_t y, uint32_t s) {
    uint32_t h = x * 0x9E3779B1u ^ (y * 0x85EBCA77u) ^ (s * 0xC2B2AE3Du);
    h ^= h >> 15; h *= 0x2C1B3C6Du; h ^= h >> 12; h *= 0x297A2D39u; h ^= h >> 15;
    return h;
}
static float xo_lattice(uint32_t ix, uint32_t iy, uint32_t s) {
    return (float)(xo_hash3(ix, iy, s) >> 8) * (1.0f / 8388608.0f) - 1.0f;
}
XO_EXPORT void xo_synth_terrain_f32(float *out, int64_t H, int64_t W, int64_t row0, int64_t col0,
                                    uint64_t seed64, float zmin, float zmax, int nthreads) {
    const uint32_t seed = (uint32_t)(seed64 * 0x9E3779B97F4A7C15ull >> 32);
#pragma omp parallel for num_threads(nthreads) schedule(static)
    for (int64_t y = 0; y < H; ++y) {
        const int64_t gy = y + row0;
        for (int64_t x = 0; x < W; ++x) {
            const int64_t gx = x + col0;
            float acc = 0.f, norm = 0.f;
            for (int o = 0; o < 12; ++o) {
                const int shift = 12 - o;
                const float amp = exp2f(0.8f * (float)(shift - 12));
                const int64_t cx = gx >> shift, cy = gy >> shift;
                const float inv = 1.0f / (float)(1 << shift);
                float fx = (float)(gx - (cx << shift)) * inv, fy = (float)(gy - (cy << shift)) * inv;
                fx = fx * fx * (3.f - 2.f * fx);
                fy = fy * fy * (3.f - 2.f * fy);
                const uint32_t s = seed + 0x632BE5ABu * (uint32_t)o;
                const float v00 = xo_lattice((uint32_t)cx, (uint32_t)cy, s), v10 = xo_lattice((uint32_t)cx + 1, (uint32_t)cy, s);
                const float v01 = xo_lattice((uint32_t)cx, (uint32_t)cy + 1, s), v11 = xo_lattice((uint32_t)cx + 1, (uint32_t)cy + 1, s);
                const float a = v00 + (v10 - v00) * fx, b = v01 + (v11 - v01) * fx;
                acc += amp * (a + (b - a) * fy);
                norm += amp;
            }
            float t = 0.5f + 0.5f * acc / norm * 1.8f;
            t = fminf(fmaxf(t, 0.f), 1.f);
            out[y * W + x] = zmin + (zmax - zmin) * t;
        }
    }
}

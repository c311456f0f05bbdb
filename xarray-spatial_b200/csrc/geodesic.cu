// geodesic.cu -- slope / aspect with method='geodesic' (geodesic.py:40-231, slope.py:167-264):
// every 3x3 neighbourhood goes (lat, lon, h) -> ECEF -> local East/North/Up frame of the centre
// cell, gets the curvature correction u += (e^2 + n^2) / (2 R) and a centred least-squares plane
// u = A e + B n; slope = atan(|(A, B)|), aspect = atan2(-A, -B).  All float64, float32 output.
//
// Regular grids (1-D lat per row, 1-D lon per column -- the common case, utils.py:644-649) first
// build two small trig tables (sin/cos lat and the prime-vertical radius N per row, sin/cos lon and
// of the step to the next column per column), so a cell needs no transcendental except the final
// atan / atan2, and the ECEF -> East/North/Up rotation is folded algebraically (see the kernel):
// ~230 FP64 operations per cell, FP64-bound.  Curvilinear grids (2-D lat/lon) evaluate the trig per
// neighbour.  One thread per output cell; the 27 loads hit L1/L2.
#include <math.h>

#include "common.cuh"

namespace xrs {

constexpr double kA2 = 6378137.0 * 6378137.0;
constexpr double kB2 = 6356752.314245 * 6356752.314245;
constexpr double kInv2R = 1.0 / (2.0 * 6370994.884953014);  // geodesic.py:183
constexpr double kDeg2Rad = 3.141592653589793 / 180.0;
constexpr double kRad2Deg = 180.0 / 3.141592653589793;

struct RowTrig { double s, c, n, m; };     // sin(lat), cos(lat), N(lat), (b^2 / a^2) N(lat)
struct ColTrig { double s, c, sd, cd; };   // sin(lon), cos(lon), sin / cos of (lon[x+1] - lon[x])

__global__ void geo_tables_kernel(const double *lat, const double *lon, int64_t H, int64_t W, RowTrig *rt,
                                  ColTrig *ct) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < H) {
        const double r = lat[i] * kDeg2Rad, s = sin(r), c = cos(r);
        rt[i].s = s; rt[i].c = c;
        const double nn = kA2 / sqrt(kA2 * c * c + kB2 * s * s);
        rt[i].n = nn;
        rt[i].m = kB2 / kA2 * nn;
    }
    if (i < W) {
        const double r = lon[i] * kDeg2Rad;
        ct[i].s = sin(r); ct[i].c = cos(r);
        const double d = (i + 1 < W) ? (lon[i + 1] - lon[i]) * kDeg2Rad : 0.0;
        ct[i].sd = sin(d); ct[i].cd = cos(d);
    }
}

struct GeoArgs {
    const void *elev;
    int64_t pitch_elems;
    const double *lat, *lon;     // 2-D mode: (H, W) contiguous; 1-D mode: unused
    const RowTrig *rt;
    const ColTrig *ct;
    float *out;
    int64_t out_pitch_elems;
    int64_t H, W;
    double z_factor;
    int want_aspect;
};

template <typename TE, bool GRID2D>
__global__ void __launch_bounds__(256) geodesic_kernel(const __grid_constant__ GeoArgs a) {
    const TE *elev = reinterpret_cast<const TE *>(a.elev);
    const int64_t n = a.H * a.W;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t y = i / a.W, x = i % a.W;
        float res = nan_of<float>();
        if (y >= 1 && y < a.H - 1 && x >= 1 && x < a.W - 1) {
            double h9[9];
            bool ok = true;
#pragma unroll
            for (int dy = 0; dy < 3; ++dy)
#pragma unroll
                for (int dx = 0; dx < 3; ++dx) {
                    const double v = (double)elev[(y + dy - 1) * a.pitch_elems + x + dx - 1];
                    h9[dy * 3 + dx] = v;
                    ok = ok && (v == v);
                }
            if (ok) {
                double Se = 0.0, Sn = 0.0, Su = 0.0, See = 0.0, Snn = 0.0, Sen = 0.0, Seu = 0.0, Snu = 0.0;
                if constexpr (!GRID2D) {
                    // Regular grid.  With t = (N + h) cos(lat), Z = (b^2/a^2 N + h) sin(lat) and
                    // D = lon_k - lon_c, rotating the ECEF offset into the centre's frame collapses to
                    //   e = t_k sin D,  p = t_k cos D - t_c,  w = Z_k - Z_c,
                    //   n = cos(lat_c) w - sin(lat_c) p,  u = cos(lat_c) p + sin(lat_c) w
                    // (the same quantities as geodesic.py:60-118 forms through X, Y, Z: ~23 FP64
                    // operations per neighbour instead of ~36, none for e in the centre's column).
                    const RowTrig rows[3] = {a.rt[y - 1], a.rt[y], a.rt[y + 1]};
                    const ColTrig cl = a.ct[x - 1], cm = a.ct[x];
                    const double sdl = -cl.sd, cdl = cl.cd, sdr = cm.sd, cdr = cm.cd;
                    const double sc = rows[1].s, cc_ = rows[1].c;
                    const double hc = h9[4] * a.z_factor;
                    const double tc = (rows[1].n + hc) * cc_, Zc = (rows[1].m + hc) * sc;
#pragma unroll
                    for (int k = 0; k < 9; ++k) {
                        if (k == 4) continue;  // the centre contributes e = n = u = 0
                        const RowTrig &r = rows[k / 3];
                        const int dxk = k % 3;
                        const double h = h9[k] * a.z_factor;
                        const double t = (r.n + h) * r.c, Z = (r.m + h) * r.s;
                        const double q = dxk == 1 ? t : t * (dxk == 0 ? cdl : cdr);
                        const double pk = q - tc, wk = Z - Zc;
                        const double nk = fma(cc_, wk, -(sc * pk));
                        double uk = fma(cc_, pk, sc * wk);
                        if (dxk == 1) {
                            uk = fma(nk * nk, kInv2R, uk);
                        } else {
                            const double ek = t * (dxk == 0 ? sdl : sdr);
                            uk = fma(fma(ek, ek, nk * nk), kInv2R, uk);
                            Se += ek;
                            See = fma(ek, ek, See); Sen = fma(ek, nk, Sen); Seu = fma(ek, uk, Seu);
                        }
                        Sn += nk; Su += uk;
                        Snn = fma(nk, nk, Snn); Snu = fma(nk, uk, Snu);
                    }
                } else {
                // centre cell first (it defines the local frame), then one neighbour at a time:
                // ECEF -> offset -> (e, n, u) -> running sums of the normal equations.  The sums are
                // accumulated uncentred and centred at the end (sum(de*du) = sum(e*u) - 9*me*mu);
                // e and n are symmetric about 0 within a 3x3 window, so nothing cancels badly.
                RowTrig rc;
                ColTrig cc;
                auto trig = [&](int dy, int dx, RowTrig &r, ColTrig &c) {
                    const int64_t j = (y + dy - 1) * a.W + x + dx - 1;
                    const double la = a.lat[j] * kDeg2Rad, lo = a.lon[j] * kDeg2Rad;
                    r.s = sin(la); r.c = cos(la);
                    r.n = kA2 / sqrt(kA2 * r.c * r.c + kB2 * r.s * r.s);
                    c.s = sin(lo); c.c = cos(lo);
                };
                auto ecef = [&](const RowTrig &r, const ColTrig &c, double h, double &X, double &Y, double &Z) {
                    const double t = (r.n + h) * r.c;
                    X = t * c.c;
                    Y = t * c.s;
                    Z = (kB2 / kA2 * r.n + h) * r.s;
                };
                trig(1, 1, rc, cc);
                double Xc, Yc, Zc;
                ecef(rc, cc, h9[4] * a.z_factor, Xc, Yc, Zc);
                const double ex = -cc.s, ey = cc.c;
                const double nx = -rc.s * cc.c, ny = -rc.s * cc.s, nz = rc.c;
                const double ux = rc.c * cc.c, uy = rc.c * cc.s, uz = rc.s;
#pragma unroll
                for (int k = 0; k < 9; ++k) {
                    if (k == 4) continue;  // the centre contributes e = n = u = 0
                    RowTrig r;
                    ColTrig c;
                    trig(k / 3, k % 3, r, c);
                    double Xk, Yk, Zk;
                    ecef(r, c, h9[k] * a.z_factor, Xk, Yk, Zk);
                    const double dx = Xk - Xc, dy = Yk - Yc, dz = Zk - Zc;
                    const double ek = dx * ex + dy * ey;  // ez = 0
                    const double nk = dx * nx + dy * ny + dz * nz;
                    double uk = dx * ux + dy * uy + dz * uz;
                    uk += (ek * ek + nk * nk) * kInv2R;
                    Se += ek; Sn += nk; Su += uk;
                    See = fma(ek, ek, See); Snn = fma(nk, nk, Snn); Sen = fma(ek, nk, Sen);
                    Seu = fma(ek, uk, Seu); Snu = fma(nk, uk, Snu);
                }
                }
                const double me = Se * (1.0 / 9.0), mn = Sn * (1.0 / 9.0), mu = Su * (1.0 / 9.0);
                See -= 9.0 * me * me; Snn -= 9.0 * mn * mn; Sen -= 9.0 * me * mn;
                Seu -= 9.0 * me * mu; Snu -= 9.0 * mn * mu;
                const double det = See * Snn - Sen * Sen;
                double A = 0.0, B = 0.0;
                if (!(fabs(det) < 1e-30)) {
                    const double inv = 1.0 / det;
                    A = (Seu * Snn - Snu * Sen) * inv;
                    B = (Snu * See - Seu * Sen) * inv;
                }
                // A, B are float64; the result is float32, so the transcendental tail runs in
                // float32 (one MUFU + a degree-7 polynomial, 2.5e-7 relative) like the planar path
                const double m2 = A * A + B * B;
                if (!a.want_aspect) {
                    res = atan_sqrt_deg((float)m2);
                } else if (m2 < 1e-14) {   // |(A, B)| < 1e-7 (geodesic.py:160)
                    res = -1.0f;
                } else {
                    res = compass_deg((float)(-A), (float)(-B));   // atan2(-A, -B) folded to [0, 360)
                }
            }
        }
        a.out[y * a.out_pitch_elems + x] = res;
    }
}

}  // namespace xrs

using namespace xrs;

extern "C" int xrs_geodesic(const void *elev, int elev_dtype, int64_t elev_pitch, const double *lat,
                            const double *lon, int latlon_2d, float *out, int64_t out_pitch, int64_t H, int64_t W,
                            double z_factor, int want_aspect, xrs_stream_t s) {
    if (H <= 0 || W <= 0) return XRS_OK;
    XRS_REQUIRE(elev_dtype == XRS_F32 || elev_dtype == XRS_F64, "elevation must be float32 or float64");
    XRS_TRY(check_cells_arg(elev, elev_dtype, kRasterCells, elev_pitch, W));
    XRS_REQUIRE(lat && lon && out, "NULL pointer");
    XRS_TRY(check_out_pitch(out_pitch, 4, W));
    const int esz = cell_size(elev_dtype);
    cudaStream_t st = (cudaStream_t)s;
    GeoArgs a;
    a.elev = elev; a.pitch_elems = elev_pitch / esz; a.lat = lat; a.lon = lon; a.rt = nullptr; a.ct = nullptr;
    a.out = out; a.out_pitch_elems = out_pitch / 4; a.H = H; a.W = W; a.z_factor = z_factor;
    a.want_aspect = want_aspect;
    void *scratch = nullptr;
    if (!latlon_2d) {
        XRS_CUDA(cudaMallocAsync(&scratch, (size_t)H * sizeof(RowTrig) + (size_t)W * sizeof(ColTrig), st));
        RowTrig *rt = (RowTrig *)scratch;
        ColTrig *ct = (ColTrig *)(rt + H);
        const int64_t m = H > W ? H : W;
        geo_tables_kernel<<<(unsigned)((m + 255) / 256), 256, 0, st>>>(lat, lon, H, W, rt, ct);
        a.rt = rt; a.ct = ct;
    }
    const int64_t grid = stride_grid(H * W);
    if (elev_dtype == XRS_F32) {
        if (latlon_2d) geodesic_kernel<float, true><<<(unsigned)grid, 256, 0, st>>>(a);
        else geodesic_kernel<float, false><<<(unsigned)grid, 256, 0, st>>>(a);
    } else {
        if (latlon_2d) geodesic_kernel<double, true><<<(unsigned)grid, 256, 0, st>>>(a);
        else geodesic_kernel<double, false><<<(unsigned)grid, 256, 0, st>>>(a);
    }
    cudaError_t e = cudaGetLastError();
    if (scratch) cudaFreeAsync(scratch, st);
    if (e != cudaSuccess) return cuda_fail(e, "geodesic_kernel launch");
    return XRS_OK;
}

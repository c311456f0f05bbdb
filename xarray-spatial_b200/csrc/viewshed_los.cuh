// viewshed_los.cuh -- viewshed (viewshed.py:1122-1502 of the reference) as a per-cell line-of-sight test.
// Everything here is __host__ __device__ and free of CUDA calls, so the CPU tests compile this header with g++
// and run the same steps as the kernels (viewshed.cu); both builds keep FMA contraction off.
//
// The reference sweeps the cells' ENTER / CENTER / EXIT events by angle around the observer through a red-black
// tree keyed by the squared distance.  Its answer for a cell t depends only on which cells are in the tree when
// t's CENTER event is handled, so each cell can decide on its own (DESIGN.md section 4.8):
//
//   node(c)  angles A0, A1, A2 of c's ENTER corner, centre and EXIT corner (row / column index units) and the
//            gradients G0, G1, G2 = atan((elev - vp_elev) / dist) at those points (coordinate units); the corner
//            elevations are the mean of the 4 cells around the corner, or c's own value.
//   t is visible  iff  no blocker c has g_c(A1(t)) > G1'(t), where G1'(t) uses z(t) + target_elev, g_c is the
//            reference's linear interpolation through (A0, G0), (A1, G1), (A2, G2), and a blocker is any c with
//            key(c) < key(t) whose event interval holds A1(t) strictly: A0 < A1(t) < A2.  Events are sorted by
//            angle, then EXIT < CENTER < ENTER, which makes the interval open.
//   wrap     cells in the observer's row east of it (A0 > A1 = 0) are in the tree from the start until their EXIT,
//            as (A0 - 2 pi, 0, A2), and again after their ENTER near 2 pi, as (A0, 2 pi, A2 + 2 pi).
//
// The interval of c is the angular extent of its square seen from the observer centre, so the blockers of t are
// among the cells the segment observer -> t crosses; for_each_candidate() walks those along the major axis with
// a margin, and the exact tests above decide.  Cells past t along the major axis have key > key(t).
#pragma once
#include <math.h>
#include <stdint.h>

#ifndef __CUDACC__
#define __host__
#define __device__
#endif

namespace xrs {
namespace vs {

constexpr double kPi = 3.141592653589793;   // math.pi

// fdlibm's atan (argument reduction at 7/16, 11/16, 19/16, 39/16 and a degree-22 odd polynomial), written with
// + - * / only so the GPU and the host round identically; within one ulp of the true value.
__host__ __device__ inline double atan64(double x) {
    const double aT[11] = {3.33333333333329318027e-01, -1.99999999998764832476e-01, 1.42857142725034663711e-01,
                           -1.11111104054623557880e-01, 9.09088713343650656196e-02, -7.69187620504482999495e-02,
                           6.66107313738753120669e-02, -5.83357013379057348645e-02, 4.97687799461593236017e-02,
                           -3.65315727442169155270e-02, 1.62858201153657823623e-02};
    if (x != x) return x + x;
    const bool neg = x < 0.0;
    double a = neg ? -x : x;
    if (a >= 7.3786976294838206464e19) {   // 2^66
        const double r = 1.57079632679489655800e+00 + 6.12323399573676603587e-17;
        return neg ? -r : r;
    }
    int id;
    if (a < 0.4375) {
        if (a < 7.450580596923828125e-9) return x;   // 2^-27
        id = -1;
        a = x;
    } else if (a < 1.1875) {
        if (a < 0.6875) { id = 0; a = (2.0 * a - 1.0) / (2.0 + a); }
        else { id = 1; a = (a - 1.0) / (a + 1.0); }
    } else if (a < 2.4375) {
        id = 2; a = (a - 1.5) / (1.0 + 1.5 * a);
    } else {
        id = 3; a = -1.0 / a;
    }
    const double z = a * a, w = z * z;
    const double s1 = z * (aT[0] + w * (aT[2] + w * (aT[4] + w * (aT[6] + w * (aT[8] + w * aT[10])))));
    const double s2 = w * (aT[1] + w * (aT[3] + w * (aT[5] + w * (aT[7] + w * aT[9]))));
    if (id < 0) return a - a * (s1 + s2);
    // atan(0.5), atan(1), atan(1.5), atan(inf) split into high and low parts
    const double hi = id == 0 ? 4.63647609000806093515e-01 : id == 1 ? 7.85398163397448278999e-01
                    : id == 2 ? 9.82793723247329054082e-01 : 1.57079632679489655800e+00;
    const double lo = id == 0 ? 2.26987774529616870924e-17 : id == 1 ? 3.06161699786838301793e-17
                    : id == 2 ? 1.39033110312309984516e-17 : 6.12323399573676603587e-17;
    const double r = hi - ((a * (s1 + s2) - lo) - a);
    return neg ? -r : r;
}

enum Event { kExit = -1, kCenter = 0, kEnter = 1 };

struct Node {           // 56 bytes per cell in the node table
    double a0, a1, a2;  // ENTER, centre and EXIT angles, raw (unshifted)
    double g0, g1, g2;  // gradients at the ENTER corner, centre and EXIT corner
    double zt;          // z + target_elev: the cell seen as a target
};

struct View {
    int64_t H, W, vr, vc;        // raster shape and observer cell
    double vp_elev, target, ew, ns;

    // squared distance of cell (r, c) in coordinate units (_calc_dist_n_grad)
    __host__ __device__ double key(int64_t r, int64_t c) const {
        const double dx = (double)(c - vc) * ew, dy = (double)(r - vr) * ns;
        return dx * dx + dy * dy;
    }
    // _calc_event_grad: the gradient of elevation `elev` seen at index position (y, x)
    __host__ __device__ double grad(double y, double x, double elev) const {
        const double diff = elev - vp_elev;
        const double dx = (x - (double)vc) * ew, dy = (y - (double)vr) * ns;
        const double d2 = dx * dx + dy * dy;
        if (d2 == 0.0) return diff > 0.0 ? kPi / 2 : (diff < 0.0 ? -kPi / 2 : 0.0);
        return atan64(diff / sqrt(d2));
    }
    // _calculate_angle of the index position (y, x), counter-clockwise from east with rows growing downwards
    __host__ __device__ double angle(double y, double x) const {
        const double px = (double)vc, py = (double)vr;
        if (px == x && py > y) return kPi / 2;
        if (px == x && py < y) return kPi * 3.0 / 2.0;
        if (x == px && y == py) return 0.0;
        if (py == y && x > px) return 0.0;
        if (px > x && py == y) return kPi;
        const double ang = atan64(fabs(y - py) / fabs(x - px));
        if (x > px && y < py) return ang;
        if (px > x && py > y) return kPi - ang;
        if (px > x && py < y) return kPi + ang;
        if (px < x && py < y) return kPi * 2.0 - ang;
        return 0.0;
    }
    // _calc_event_pos: the ENTER (e = +1) or EXIT (e = -1) corner of cell (r, c) as half-cell offsets (dy, dx)
    __host__ __device__ void corner(int e, int64_t r, int64_t c, int &dy, int &dx) const {
        const int sr = r < vr ? -1 : (r > vr ? 1 : 0), sc = c < vc ? -1 : (c > vc ? 1 : 0);
        if (sr < 0 && sc < 0) { dy = e > 0 ? -1 : 1; dx = e > 0 ? 1 : -1; }
        else if (sr < 0 && sc == 0) { dy = 1; dx = e > 0 ? 1 : -1; }
        else if (sr < 0 && sc > 0) { dy = e > 0 ? 1 : -1; dx = e > 0 ? 1 : -1; }
        else if (sr == 0 && sc > 0) { dy = e > 0 ? 1 : -1; dx = -1; }
        else if (sr > 0 && sc > 0) { dy = e > 0 ? 1 : -1; dx = e > 0 ? -1 : 1; }
        else if (sr > 0 && sc == 0) { dy = -1; dx = e > 0 ? -1 : 1; }
        else if (sr > 0 && sc < 0) { dy = e > 0 ? -1 : 1; dx = e > 0 ? -1 : 1; }
        else if (sr == 0 && sc < 0) { dy = e > 0 ? -1 : 1; dx = 1; }
        else { dy = 0; dx = 0; }
    }
};

// The node of cell (r, c) != observer.  Z(r, c) returns the cell's elevation as float64.
template <typename Z> __host__ __device__ inline Node make_node(const View &v, const Z &z, int64_t r, int64_t c) {
    Node n;
    const double e = z(r, c);
    for (int k = 0; k < 2; ++k) {   // _calc_event_elev of the ENTER, then the EXIT corner
        int dy, dx;
        v.corner(k == 0 ? kEnter : kExit, r, c, dy, dx);
        const int64_t r1 = r + dy, c1 = c + dx;   // the cell diagonally across the corner
        double el = e;
        if (r1 >= 0 && r1 < v.H && c1 >= 0 && c1 < v.W) {
            const double e1 = z(r1, c1), e2 = z(r1, c), e3 = z(r, c1);
            if (!(e1 != e1 || e2 != e2 || e3 != e3 || e != e)) el = (e1 + e2 + e3 + e) / 4.0;
        }
        const double y = (double)r + 0.5 * dy, x = (double)c + 0.5 * dx;
        if (k == 0) { n.a0 = v.angle(y, x); n.g0 = v.grad(y, x, el); }
        else { n.a2 = v.angle(y, x); n.g2 = v.grad(y, x, el); }
    }
    n.a1 = v.angle((double)r, (double)c);
    n.g1 = v.grad((double)r, (double)c, e);
    n.zt = e + v.target;
    return n;
}

// The gradient of the target (the CENTER event's G1', from z + target_elev).
__host__ __device__ inline double target_grad(const View &v, double key, double zt) {
    const double diff = zt - v.vp_elev;
    if (key == 0.0) return diff > 0.0 ? kPi / 2 : (diff < 0.0 ? -kPi / 2 : 0.0);
    return atan64(diff / sqrt(key));
}

// _get_vertical_ang: degrees, 0 straight below the observer, 90 level, 180 straight above
__host__ __device__ inline double vertical_angle(double vp_elev, double key, double elev) {
    const double diff = vp_elev - elev;
    if (diff == 0.0) return 90.0;
    if (diff > 0.0) return atan64(sqrt(key) / diff) * 180.0 / kPi;
    return atan64(fabs(diff) / sqrt(key)) * 180.0 / kPi + 90.0;
}

// Does node n hold angle th in the status structure?  Sets the angles it holds them with (the wrap rule).
__host__ __device__ inline bool member(const Node &n, double th, double &A0, double &A1, double &A2) {
    if (!(n.a0 > n.a1)) {
        A0 = n.a0; A1 = n.a1; A2 = n.a2;
        return n.a0 < th && th < n.a2;
    }
    if (th < n.a2) { A0 = n.a0 - 2 * kPi; A1 = n.a1; A2 = n.a2; return true; }
    if (th > n.a0) { A0 = n.a0; A1 = n.a1 + 2 * kPi; A2 = n.a2 + 2 * kPi; return true; }
    return false;
}

// The reference's interpolated gradient of a member node at angle th (viewshed.py:430-446), same operation order.
__host__ __device__ inline double interp(const Node &n, double A0, double A1, double A2, double th) {
    if (th < A1) return n.g1 + (n.g0 - n.g1) * (A1 - th) / (A1 - A0);
    if (th > A1) return n.g1 + (n.g2 - n.g1) * (th - A1) / (A2 - A1);
    return n.g1;
}

// Does member node n put gradient > gt on angle th?  The interpolation lies between its two end gradients up to
// a few ulps, so the division only runs when gt is within 1e-12 of that range.
__host__ __device__ inline bool exceeds(const Node &n, double th, double gt) {
    double A0, A1, A2;
    if (!member(n, th, A0, A1, A2)) return false;
    const double ge = th < A1 ? n.g0 : (th > A1 ? n.g2 : n.g1);
    const double lo = ge < n.g1 ? ge : n.g1, hi = ge < n.g1 ? n.g1 : ge;
    if (hi < gt - 1e-12) return false;
    if (lo > gt + 1e-12) return true;
    return interp(n, A0, A1, A2, th) > gt;
}

// Calls f(r, c) for every cell in the raster the segment from the observer to (vr + dr, vc + dc) can cross, by
// steps along the major axis up to the target's own step; f returns true to stop.  The 2^-30 margin (in cells)
// keeps rounding in the stepping from dropping a crossed cell while the raster is under 2^29 cells a side.
template <typename F> __host__ __device__ inline void for_each_candidate(const View &v, int64_t dr, int64_t dc, F &&f) {
    const bool xmaj = (dc < 0 ? -dc : dc) >= (dr < 0 ? -dr : dr);
    const int64_t maj = xmaj ? dc : dr, mnr = xmaj ? dr : dc;
    const int64_t n = maj < 0 ? -maj : maj, s = maj < 0 ? -1 : 1;
    if (n == 0) return;
    const double m = (double)mnr / (double)n;
    const double eps = 9.313225746154785e-10;
    for (int64_t u = 1; u <= n; ++u) {
        double a = ((double)u - 0.5) * m, b = ((double)u + 0.5) * m;
        if (a > b) { const double t = a; a = b; b = t; }
        const int64_t wlo = (int64_t)floor(a - 0.5 - eps) + 1, whi = (int64_t)ceil(b + 0.5 + eps) - 1;
        for (int64_t w = wlo; w <= whi; ++w) {
            const int64_t r = v.vr + (xmaj ? w : s * u), c = v.vc + (xmaj ? s * u : w);
            if (r < 0 || r >= v.H || c < 0 || c >= v.W) continue;
            if (f(r, c)) return;
        }
    }
}

// The output of cell (r, c): 180 for the observer, -1 when invisible, the vertical angle otherwise.  N(r, c)
// returns the node of a cell.
template <typename N> __host__ __device__ inline double cell_value(const View &v, const N &node, int64_t r, int64_t c) {
    if (r == v.vr && c == v.vc) return 180.0;
    const Node t = node(r, c);
    const double kt = v.key(r, c);
    const double gt = target_grad(v, kt, t.zt);
    if (!(gt == gt)) return -1.0;               // max <= NaN never holds
    const double th = t.a1;
    bool blocked = false;
    for_each_candidate(v, r - v.vr, c - v.vc, [&](int64_t rr, int64_t cc) {
        if (!(v.key(rr, cc) < kt) || (rr == v.vr && cc == v.vc)) return false;
        blocked = exceeds(node(rr, cc), th, gt);
        return blocked;
    });
    return blocked ? -1.0 : vertical_angle(v.vp_elev, kt, t.zt);
}

}  // namespace vs
}  // namespace xrs

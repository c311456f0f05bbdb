// pathfinding_grid.cuh -- the exact grid arithmetic of a_star_search (pathfinding.py:233-382 of the reference):
// path lengths as step counts, the relaxation of one cell, the walk's successor rule and the snap order.
// Everything here is __host__ __device__ and free of CUDA calls, so the CPU tests compile this header with g++
// and run the same steps as the kernels (pathfinding.cu).
//
// A path length is a pair (a, b): a orthogonal and b diagonal steps, worth a + b sqrt(2).  sqrt(2) is irrational,
// so two lengths are equal exactly when their pairs are, and less() decides the order in integers.  A path has
// fewer than H W steps and H W < 2^31, so a, b and the squares in less() fit their types.
#pragma once
#include <stdint.h>

#ifndef __CUDACC__
#define __host__
#define __device__
#endif

namespace xrs {
namespace pf {

constexpr int64_t kMaxCells = (int64_t)1 << 31;   // H W must be below this
constexpr double kSqrt2 = 1.4142135623730951;     // np.sqrt(2), the length of a diagonal move
constexpr int32_t kUnreached = INT32_MAX;          // a of a cell no path reaches

struct alignas(8) Dist {
    int32_t a, b;   // orthogonal steps, diagonal steps
};

__host__ __device__ inline Dist unreached() { return Dist{kUnreached, 0}; }
__host__ __device__ inline bool reached(Dist d) { return d.a != kUnreached; }
__host__ __device__ inline bool same(Dist x, Dist y) { return x.a == y.a && x.b == y.b; }

// x < y, exactly: a1 + b1 r < a2 + b2 r  <=>  da < db r  with da = a1 - a2, db = b2 - b1, r = sqrt(2).  Decided by
// the signs, then by da^2 against 2 db^2.  An unreached length is above every reached one.
__host__ __device__ inline bool less(Dist x, Dist y) {
    if (!reached(y)) return reached(x);
    if (!reached(x)) return false;
    const int64_t da = (int64_t)x.a - y.a, db = (int64_t)y.b - x.b;
    const uint64_t da2 = (uint64_t)(da * da), db2x2 = 2 * (uint64_t)(db * db);
    if (db > 0) return da < 0 || da2 < db2x2;
    if (da >= 0) return false;
    return db == 0 || da2 > db2x2;   // both negative: |da| > |db| r
}

// The reference's neighbour order (_neighborhood_structure): move k of connectivity 8 or 4 as (dy, dx).
__host__ __device__ inline int n_moves(int conn) { return conn == 8 ? 8 : 4; }
__host__ __device__ inline void move(int conn, int k, int &dy, int &dx) {
    if (conn == 8) {
        dx = k < 3 ? -1 : k < 5 ? 0 : 1;
        dy = (k == 0 || k == 3 || k == 5) ? -1 : (k == 1 || k == 6) ? 0 : 1;
    } else {
        dy = k == 1 ? -1 : k == 2 ? 1 : 0;
        dx = k == 0 ? -1 : k == 3 ? 1 : 0;
    }
}

// d plus one move: (1, 0) orthogonal, (0, 1) diagonal.
__host__ __device__ inline Dist add_step(Dist d, bool diag) {
    if (!reached(d)) return d;
    return diag ? Dist{d.a, d.b + 1} : Dist{d.a + 1, d.b};
}

// One relaxation of a crossable cell holding d: the least of d and every neighbour's length plus its move.
// at(dy, dx) returns a neighbour's length, unreached() when it is outside the raster or not crossable.
template <class At> __host__ __device__ inline Dist relax(Dist d, int conn, const At &at) {
    for (int k = 0; k < n_moves(conn); ++k) {
        int dy, dx;
        move(conn, k, dy, dx);
        const Dist c = add_step(at(dy, dx), dy != 0 && dx != 0);
        if (less(c, d)) d = c;
    }
    return d;
}

// The walk's rule on the exact field of lengths to the goal: from a cell at d, the first move in the reference's
// neighbour order to a neighbour at exactly d less that move; -1 when none is (d is not the field's value).
template <class At> __host__ __device__ inline int successor(Dist d, int conn, const At &at) {
    for (int k = 0; k < n_moves(conn); ++k) {
        int dy, dx;
        move(conn, k, dy, dx);
        const Dist n = at(dy, dx);
        if (reached(n) && same(add_step(n, dy != 0 && dx != 0), d)) return k;
    }
    return -1;
}

// The running sum the reference writes along a path: d_prev + sqrt(dx^2 + dy^2) in float64.
__host__ __device__ inline double path_value(double prev, bool diag) { return prev + (diag ? kSqrt2 : 1.0); }

// _find_nearest_pixel's order, exactly: a crossable cell snaps to itself; otherwise to the crossable cell with the
// least squared pixel distance, the first in row-major order among equals, taken only below the squared diagonal
// (the reference starts from the diagonal with a strict <).
__host__ __device__ inline int64_t snap_d2(int64_t r, int64_t c, int64_t r0, int64_t c0) {
    return (r - r0) * (r - r0) + (c - c0) * (c - c0);
}
__host__ __device__ inline bool snap_qualifies(int64_t d2, int64_t H, int64_t W) {
    return d2 == 0 || d2 < (H - 1) * (H - 1) + (W - 1) * (W - 1);   // d2 == 0: the cell itself, crossable
}

}  // namespace pf
}  // namespace xrs

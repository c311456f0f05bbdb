// proximity_envelope.cuh -- the column pass of the exact nearest-target transform (proximity.cu), for one
// column of the raster: build each band's envelope, merge the bands' envelopes, walk the merged envelope for
// every query row.  Everything here is __host__ __device__ and free of CUDA calls, so the CPU tests compile this
// header with g++ and run the same steps as the kernels.
//
// Every row r that holds a target carries one candidate for column c: the target the row pass picked in row r
// (ridx[r][c]).  Its cost at query row i is the metric's distance key between cell (i, c) and that target; the
// column pass finds, for every i, the row whose candidate costs least, the earliest row on a tie.  Each metric
// gives the candidates a position u (ascending with the row index) and a parameter v:
//   Euclidean     u = Y'_r, v = dx^2                  cost = v + (Y_i - Y_r)^2     (lower envelope of parabolas)
//   Manhattan     u = Y'_r, v = |dx|                  cost = v + |Y_i - Y_r|       (lower envelope of V shapes)
//   great circle  u = sin(lat_r), v = cos(lat_r) cos(dlon)
//                                                     cost = -(cos(lat_i) v + sin(lat_i) sin(lat_r))
// (Y' and sin(lat) are negated when the coordinate descends, so u always ascends.)  For the great circle, the
// cost is the chord's -(1 - chord^2 / 2): the nearest row is the support point of the points (v, u) in the
// direction (cos lat_i, sin lat_i), i.e. the right hull chain of points sorted by u.
//
// For two candidates q before r, the cost difference f_q - f_r never decreases as the query moves down the
// column, so q wins (ties included) on a prefix of the queries and r on the rest.  q leaves the envelope when its
// winning range against its successor ends no later than its predecessor's against it (pop()); the tests are
// division-free, so integer-spaced grids decide ties exactly.
#pragma once
#include <math.h>
#include <stdint.h>

#ifndef __CUDACC__
#define __host__
#define __device__
#endif

namespace xrs {
namespace prox {

enum Metric { kEuclidean = 0, kGreatCircle = 1, kManhattan = 2 };   // the reference's metric ids

struct Cand {
    double u, v;
};

// 2 x the last query position where q (before r) still costs no more than r; +-inf when that is never / always.
__host__ __device__ inline double manhattan_split(Cand q, Cand r) {
    if ((q.v - q.u) - (r.v - r.u) <= 0.0) return INFINITY;   // q's right arm at or below r's: q never loses
    if ((q.u + q.v) - (r.u + r.v) > 0.0) return -INFINITY;   // q's left arm above r's: q never wins
    return (r.u + r.v) - (q.v - q.u);
}

// True when q, between p and r, is the strict winner at no query position: it leaves the envelope.
template <int M> __host__ __device__ inline bool pop(Cand p, Cand q, Cand r) {
    if (M == kEuclidean) {
        const double dpq = q.u - p.u, dqr = r.u - q.u;
        return (r.u - p.u) * dqr * dpq + (r.v - q.v) * dpq - (q.v - p.v) * dqr <= 0.0;
    } else if (M == kManhattan) {
        return manhattan_split(q, r) <= manhattan_split(p, q);
    } else {   // right hull chain of the points (v, u): q is not strictly right of the segment p -> r
        return (q.v - p.v) * (r.u - q.u) <= (r.v - q.v) * (q.u - p.u);
    }
}

// One column of the scratch.  Arrays are row-major with a stride of W between rows (band arrays: between bands).
template <int M> struct Column {
    const int32_t *ridx;   // [H][W] row pass: target column picked in each row, -1 when the row has none
    int32_t *stk;          // [H][W] envelope slots: band b's local envelope at rows b*band_rows ...
    int32_t *blo, *bhi;    // [nb][W] band b's surviving slice [lo, hi) of its local envelope
    int32_t *bprev;        // [nb][W] the band holding the envelope element below band b's first one, -1 for none
    int32_t *boff;         // [nb + 1][W] envelope elements before band b's slice; boff[nb] = envelope size
    const double *X, *Y;   // coordinates of the columns / rows
    const double *cosl, *sinl, *lam;   // great circle: cos / sin of every row's latitude, longitude in radians
    int64_t H, W, c, band_rows;
    int nb;

    // +1 when the row coordinate ascends, -1 when it descends
    __host__ __device__ double sgn() const { return H > 1 && Y[H - 1] < Y[0] ? -1.0 : 1.0; }

    __host__ __device__ int32_t target(int64_t r) const { return ridx[r * W + c]; }
    __host__ __device__ int32_t &slot(int64_t s) const { return stk[s * W + c]; }
    __host__ __device__ int32_t &lo(int b) const { return blo[b * W + c]; }
    __host__ __device__ int32_t &hi(int b) const { return bhi[b * W + c]; }
    __host__ __device__ int32_t &prev(int b) const { return bprev[b * W + c]; }
    __host__ __device__ int32_t &off(int b) const { return boff[b * W + c]; }

    __host__ __device__ Cand cand(int64_t r) const {
        const int32_t t = target(r);
        if (M == kGreatCircle) return Cand{sgn() * sinl[r], cosl[r] * cos(lam[t] - lam[c])};
        const double dx = X[t] - X[c];
        return Cand{sgn() * (Y[r] - Y[0]), M == kEuclidean ? dx * dx : fabs(dx)};
    }
    // cost of row r's candidate (parameter v) at query row i
    __host__ __device__ double cost(int64_t r, double v, int64_t i) const {
        if (M == kGreatCircle) return -(cosl[i] * v + sinl[i] * sinl[r]);
        const double dy = Y[r] - Y[i];
        return M == kEuclidean ? v + dy * dy : v + fabs(dy);
    }
};

// Phase 1: band b's envelope over its own rows, in slots b*band_rows ...; returns its size (also in hi(b)).
template <int M> __host__ __device__ inline int build_band(const Column<M> &col, int b) {
    const int64_t H = col.H;
    const int64_t b0 = (int64_t)b * col.band_rows;
    const int64_t b1 = b0 + col.band_rows < H ? b0 + col.band_rows : H;
    int n = 0;
    Cand top{0.0, 0.0}, sec{0.0, 0.0};
    for (int64_t r = b0; r < b1; ++r) {
        if (col.target(r) < 0) continue;
        const Cand cr = col.cand(r);
        while (n >= 2 && pop<M>(sec, top, cr)) {
            --n;
            top = sec;
            if (n >= 2) sec = col.cand(col.slot(b0 + n - 2));
        }
        col.slot(b0 + n) = (int32_t)r;
        ++n;
        sec = top;
        top = cr;
    }
    col.lo(b) = 0;
    col.hi(b) = n;
    return n;
}

// Phase 2: merges the bands' envelopes in order into one envelope of the whole column, kept as each band's
// surviving slice [lo, hi) of its local envelope.  Band b's elements can only be popped from the front of its
// slice while b is merged (an element whose local predecessor is still below it passed this very test in
// build_band), and from the back by later bands, so a slice stays contiguous.  Returns the envelope's size.
template <int M> __host__ __device__ inline int merge_bands(const Column<M> &col) {
    int tb = -1;                 // band of the top element
    Cand top{0.0, 0.0}, sec{0.0, 0.0};
    bool has_sec = false;
    for (int b = 0; b < col.nb; ++b) {
        const int n = col.hi(b);
        const int64_t base = (int64_t)b * col.band_rows;
        col.lo(b) = 0;
        col.hi(b) = 0;           // empty until its first element is pushed
        int j = 0;
        for (; j < n; ++j) {
            if (tb == b && j >= col.lo(b) + 2) break;   // the rest keep their local neighbours: no more pops
            const Cand cr = col.cand(col.slot(base + j));
            while (has_sec && pop<M>(sec, top, cr)) {
                --col.hi(tb);
                if (col.hi(tb) == col.lo(tb)) tb = col.prev(tb);
                top = sec;
                // the element below the new top
                int sb = tb, sp = col.hi(tb) - 2;
                if (sp < col.lo(sb)) {
                    sb = col.prev(sb);
                    sp = sb >= 0 ? col.hi(sb) - 1 : -1;
                }
                has_sec = sb >= 0;
                if (has_sec) sec = col.cand(col.slot((int64_t)sb * col.band_rows + sp));
            }
            if (tb != b) {       // b's slice starts here
                col.prev(b) = tb;
                col.lo(b) = j;
                tb = b;
            }
            col.hi(b) = j + 1;
            has_sec = (col.hi(b) - col.lo(b) >= 2) || col.prev(b) >= 0;
            sec = top;
            top = cr;
        }
        if (j < n) {
            col.hi(b) = n;
            top = col.cand(col.slot(base + n - 1));
            sec = col.cand(col.slot(base + n - 2));
            has_sec = true;
        }
    }
    int total = 0;
    for (int b = 0; b < col.nb; ++b) {
        col.off(b) = total;
        total += col.hi(b) - col.lo(b);
    }
    col.off(col.nb) = total;
    return total;
}

// An element of the merged envelope: its band, index in the band's local envelope, row and parameter.
template <int M> struct Cursor {
    int band, pos;
    int64_t row;
    double v;
};

template <int M> __host__ __device__ inline void cursor_load(const Column<M> &col, Cursor<M> &k) {
    k.row = col.slot((int64_t)k.band * col.band_rows + k.pos);
    k.v = col.cand(k.row).v;
}

// The element with global index k (0 <= k < envelope size).
template <int M> __host__ __device__ inline Cursor<M> cursor_at(const Column<M> &col, int k) {
    int a = 0, z = col.nb - 1;   // the last band whose offset is <= k holds it
    while (a < z) {
        const int m = (a + z + 1) >> 1;
        if (col.off(m) <= k) a = m; else z = m - 1;
    }
    Cursor<M> e;
    e.band = a;
    e.pos = col.lo(a) + (k - col.off(a));
    cursor_load(col, e);
    return e;
}

template <int M> __host__ __device__ inline bool cursor_next(const Column<M> &col, const Cursor<M> &k,
                                                               Cursor<M> &n) {
    n.band = k.band;
    n.pos = k.pos + 1;
    while (n.pos >= col.hi(n.band)) {
        if (++n.band >= col.nb) return false;
        n.pos = col.lo(n.band);
    }
    cursor_load(col, n);
    return true;
}

// Phase 3: for every query row of band b, the row of the nearest candidate (earliest on a tie), or -1 when the
// column has none; calls emit(i, row).  The start is a binary search at the band's first row, then a walk.
template <int M, typename Emit> __host__ __device__ inline void query_band(const Column<M> &col, int b, Emit &&emit) {
    const int64_t H = col.H;
    const int64_t b0 = (int64_t)b * col.band_rows;
    const int64_t b1 = b0 + col.band_rows < H ? b0 + col.band_rows : H;
    const int total = col.off(col.nb);
    if (total == 0) {
        for (int64_t i = b0; i < b1; ++i) emit(i, (int64_t)-1);
        return;
    }
    int a = 0, z = total - 1;    // first k whose successor is not strictly cheaper at row b0
    while (a < z) {
        const int m = (a + z) >> 1;
        const Cursor<M> e = cursor_at(col, m), f = cursor_at(col, m + 1);
        if (col.cost(f.row, f.v, b0) < col.cost(e.row, e.v, b0)) a = m + 1; else z = m;
    }
    Cursor<M> cur = cursor_at(col, a), nxt;
    bool more = cursor_next(col, cur, nxt);
    for (int64_t i = b0; i < b1; ++i) {
        while (more && col.cost(nxt.row, nxt.v, i) < col.cost(cur.row, cur.v, i)) {
            cur = nxt;
            more = cursor_next(col, cur, nxt);
        }
        emit(i, cur.row);
    }
}

}  // namespace prox
}  // namespace xrs

// noise_octave.cuh -- the exact arithmetic of perlin (perlin.py:189) and generate_terrain (terrain.py:183): NumPy's
// legacy permutation (MT19937 and its masked-rejection draw, from mt19937.cuh), the reservation rule of the
// parallel Knuth shuffle, and one octave of the reference's NumPy noise.  Everything here is __host__ __device__
// and free of CUDA calls, so the CPU tests compile this header with g++ and run the same steps as the kernels
// (noise.cu).
//
// RandomState(seed).permutation(n) is init_genrand(seed), then Fisher-Yates from i = n - 1 down to 1: step i draws
// tempered MT19937 words w until (w & mask(i)) <= i, mask(i) being i with every lower bit set, and swaps
// A[i] with A[w & mask(i)].
#pragma once
#include <math.h>
#include <stdint.h>

#include "mt19937.cuh"

namespace xrs {
namespace nz {

using namespace mt;   // the generator and the masked-rejection draw

constexpr int64_t kTableN = (int64_t)1 << 20;   // the reference's table: permutation(2**20)
constexpr int64_t kIndexLimit = 2 * kTableN;    // np.append(p, p) takes indices in [-2^21, 2^21)
constexpr int kTerrainOctaves = 16;

// The deterministic reservations of the parallel Knuth shuffle (Shun, Gu, Blelloch, Fineman and Gibbons, SODA
// 2015): in round r every pending step i writes max(key) to positions i and J[i], and commits its swap when it
// holds both.  Sequential order is descending i, so the largest pending step touching a position goes first.
__host__ __device__ inline uint64_t reservation(uint32_t round, uint32_t i) { return ((uint64_t)round << 32) | i; }

// ---------------------------------------------------------------------------------------------- one octave
// _fade as numba evaluates it: t**5, t**4 and t**3 by squaring.
__host__ __device__ inline double fade(double t) {
    const double t2 = t * t, t4 = t2 * t2;
    return 6.0 * (t4 * t) - 15.0 * t4 + 10.0 * (t2 * t);
}

__host__ __device__ inline double lerp(double a, double b, double x) { return a + x * (b - a); }

// _gradient: vectors [[0, 1], [0, -1], [1, 0], [-1, 0]][h mod 4] . (x, y), computed literally so signed zeros
// come out as there (h >= 0: a permutation entry).
__host__ __device__ inline double gradient(int32_t h, double x, double y) {
    const int k = h & 3;
    const double gx = k == 2 ? 1.0 : k == 3 ? -1.0 : 0.0, gy = k == 0 ? 1.0 : k == 1 ? -1.0 : 0.0;
    return gx * x + gy * y;
}

// What one octave needs of a column (x) and of a row (y).
struct Col {
    double xf, u;     // x - xi, fade(x - xi)
    int32_t p0, p1;   // P[xi], P[xi + 1]
};
struct Row {
    double yf, v;     // y - yi, fade(y - yi)
    int32_t yi, pad;
};

// x.astype(int) of a float32 coordinate, and whether it is usable: a column's xi and xi + 1 must index the doubled
// table; a row's yi is usable when |yi| < 2^22 (beyond it every P[.] + yi is outside the table).
__host__ __device__ inline bool col_index(float x, int32_t &xi) {
    const double t = trunc((double)x);
    const bool ok = t >= -(double)kIndexLimit && t + 1 < (double)kIndexLimit;   // NaN fails
    xi = ok ? (int32_t)t : 0;
    return ok;
}
__host__ __device__ inline bool row_index(float y, int32_t &yi) {
    const double t = trunc((double)y);
    const bool ok = t > -4.0 * kTableN && t < 4.0 * kTableN;
    yi = ok ? (int32_t)t : 0;
    return ok;
}

// P[k] of the doubled table for k in [-2^21, 2^21), k's residue otherwise (the call raises IndexError then).
__host__ __device__ inline int32_t table_at(const int32_t *P, int64_t k) { return P[k & (kTableN - 1)]; }

__host__ __device__ inline Col make_col(const int32_t *P, float x, bool &ok) {
    int32_t xi;
    ok = col_index(x, xi);
    const double xf = (double)x - (double)xi;
    return Col{xf, fade(xf), table_at(P, xi), table_at(P, (int64_t)xi + 1)};
}

__host__ __device__ inline Row make_row(float y, bool &ok) {
    int32_t yi;
    ok = row_index(y, yi);
    const double yf = (double)y - (double)yi;
    return Row{yf, fade(yf), yi, 0};
}

// _perlin at one cell: four table reads, four gradients, three lerps.
__host__ __device__ inline double octave(const int32_t *P, const Col &c, const Row &r) {
    const int64_t y0 = r.yi, y1 = (int64_t)r.yi + 1;
    const double n00 = gradient(table_at(P, c.p0 + y0), c.xf, r.yf);
    const double n01 = gradient(table_at(P, c.p0 + y1), c.xf, r.yf - 1);
    const double n11 = gradient(table_at(P, c.p1 + y1), c.xf - 1, r.yf - 1);
    const double n10 = gradient(table_at(P, c.p1 + y0), c.xf - 1, r.yf);
    return lerp(lerp(n00, n10, c.u), lerp(n01, n11, c.u), r.v);
}

// Octave o of the terrain reads coordinates float32(x 2^o) and weighs its noise by 2^-o.
__host__ __device__ inline float octave_coord(float x, int o) { return x * (float)(1 << o); }
__host__ __device__ inline double octave_weight(int o) { return 1.0 / (double)(1 << o); }

// The terrain's steps in the cell type T: h = T(double(h) + a m) per octave; then h / 1.97 (float32(1.97) for
// float32, NumPy's weak-scalar rule); then the cube, rounded once from the float64 product.
template <typename T> __host__ __device__ inline T terrain_add(T h, double a, double m) { return (T)((double)h + a * m); }
template <typename T> __host__ __device__ inline T terrain_scale(T h) { return h / (T)1.97; }
template <typename T> __host__ __device__ inline T terrain_cube(T h) {
    const double d = (double)h;
    return (T)(d * d * d);
}

}  // namespace nz
}  // namespace xrs

// noise_octave.cuh -- the exact arithmetic of perlin (perlin.py:189) and generate_terrain (terrain.py:183): NumPy's
// legacy permutation (MT19937 and its masked-rejection draw), the reservation rule of the parallel Knuth shuffle,
// and one octave of the reference's NumPy noise.  Everything here is __host__ __device__ and free of CUDA calls, so
// the CPU tests compile this header with g++ and run the same steps as the kernels (noise.cu).
//
// RandomState(seed).permutation(n) is init_genrand(seed), then Fisher-Yates from i = n - 1 down to 1: step i draws
// tempered MT19937 words w until (w & mask(i)) <= i, mask(i) being i with every lower bit set, and swaps
// A[i] with A[w & mask(i)].
#pragma once
#include <math.h>
#include <stdint.h>

#ifndef __CUDACC__
#define __host__
#define __device__
#endif

namespace xrs {
namespace nz {

constexpr int kMtN = 624, kMtM = 397;
constexpr uint32_t kMatrixA = 0x9908b0dfu, kUpper = 0x80000000u, kLower = 0x7fffffffu;
// The twist of one 624-word block in four phases.  A word of one phase reads only words of earlier phases (new
// values) or of later phases (old values), so each phase is parallel once all its reads precede its writes.
// Phase p covers words [phase_begin(p), phase_begin(p + 1)): 0-226, 227-453, 454-622, 623.
__host__ __device__ inline int phase_begin(int p) {
    return p == 0 ? 0 : p == 1 ? kMtN - kMtM : p == 2 ? 2 * (kMtN - kMtM) : p == 3 ? kMtN - 1 : kMtN;
}

constexpr int64_t kTableN = (int64_t)1 << 20;   // the reference's table: permutation(2**20)
constexpr int64_t kIndexLimit = 2 * kTableN;    // np.append(p, p) takes indices in [-2^21, 2^21)
constexpr int kTerrainOctaves = 16;

// init_genrand: NumPy's mt19937_seed for a seed in [0, 2^32 - 1].
__host__ __device__ inline void mt_init(uint32_t *mt, uint32_t seed) {
    mt[0] = seed;
    for (int i = 1; i < kMtN; ++i) mt[i] = 1812433253u * (mt[i - 1] ^ (mt[i - 1] >> 30)) + (uint32_t)i;
}

// Word k of the next block, from the state as it stands.
__host__ __device__ inline uint32_t mt_twist_word(const uint32_t *mt, int k) {
    const uint32_t y = (mt[k] & kUpper) | (mt[k + 1 == kMtN ? 0 : k + 1] & kLower);
    return mt[k + kMtM < kMtN ? k + kMtM : k + kMtM - kMtN] ^ (y >> 1) ^ ((0u - (y & 1u)) & kMatrixA);
}

__host__ __device__ inline void mt_twist(uint32_t *mt) {
    for (int k = 0; k < kMtN; ++k) mt[k] = mt_twist_word(mt, k);
}

__host__ __device__ inline uint32_t mt_temper(uint32_t y) {
    y ^= y >> 11;
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    return y ^ (y >> 18);
}

// random_interval's mask: the least 2^k - 1 >= i.
__host__ __device__ inline uint32_t interval_mask(uint32_t i) {
    i |= i >> 1;
    i |= i >> 2;
    i |= i >> 4;
    i |= i >> 8;
    return i | (i >> 16);
}

// One word of the sequential draw at step i (> 0): accepted when its masked value is at most i; then J[i] is that
// value and the next step is i - 1.
__host__ __device__ inline bool draw(uint32_t &i, uint32_t w, int32_t *J) {
    const uint32_t v = w & interval_mask(i);
    if (v > i) return false;
    J[i] = (int32_t)v;
    --i;
    return true;
}

// The chunk rule of the warp resolve: 32 consecutive words meet steps i, i - 1, ..., i - 31 at most.  When every
// step of that range has the same mask and i >= 32, a word whose masked value is at most i - 31 is accepted
// whatever the words before it did, and one above i is rejected.  Only words in between depend on their
// predecessors; a chunk holding one, or not uniform, is resolved word by word.
__host__ __device__ inline bool chunk_uniform(uint32_t i) { return i >= 32 && interval_mask(i - 31) == interval_mask(i); }
__host__ __device__ inline bool sure_accept(uint32_t v, uint32_t i) { return v <= i - 31; }
__host__ __device__ inline bool undecided(uint32_t v, uint32_t i) { return v > i - 31 && v <= i; }

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

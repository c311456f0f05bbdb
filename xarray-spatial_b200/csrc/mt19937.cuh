// mt19937.cuh -- NumPy's legacy MT19937 and what the project builds on it: the generator (init_genrand, the twist,
// the tempering), the masked-rejection draw of random_interval, and jump-ahead by a characteristic polynomial.
// The generator and the draw are __host__ __device__ and free of CUDA calls, so the CPU tests compile this header
// with g++ and run the same steps as the kernels (noise.cu, natural_breaks.cu).  The polynomial arithmetic of the
// jump is host code.
//
// Jump-ahead (Haramoto, Matsumoto, Nishimura, Panneton and L'Ecuyer, INFORMS J. Computing 2008): the generator's
// one-word step T is linear over GF(2) on the 19937-bit state, with characteristic polynomial phi.  phi is found
// once by Berlekamp-Massey on the generator's own output bits.  The state d words ahead is p(T) s with
// p = x^d mod phi, evaluated by Horner: acc = T(acc) + c_k s from the top coefficient down.
#pragma once
#include <stdint.h>

#ifndef __CUDACC__
#ifndef __host__
#define __host__
#define __device__
#endif
#endif

#include <algorithm>
#include <vector>

namespace xrs {
namespace mt {

constexpr int kMtN = 624, kMtM = 397;
constexpr int kMtBits = 19937;   // the degree of phi
constexpr uint32_t kMatrixA = 0x9908b0dfu, kUpper = 0x80000000u, kLower = 0x7fffffffu;
// The twist of one 624-word block in four phases.  A word of one phase reads only words of earlier phases (new
// values) or of later phases (old values), so each phase is parallel once all its reads precede its writes.
// Phase p covers words [phase_begin(p), phase_begin(p + 1)): 0-226, 227-453, 454-622, 623.
__host__ __device__ inline int phase_begin(int p) {
    return p == 0 ? 0 : p == 1 ? kMtN - kMtM : p == 2 ? 2 * (kMtN - kMtM) : p == 3 ? kMtN - 1 : kMtN;
}

// init_genrand: NumPy's mt19937_seed for a seed in [0, 2^32 - 1].
__host__ __device__ inline void mt_init(uint32_t *mt, uint32_t seed) {
    mt[0] = seed;
    for (int i = 1; i < kMtN; ++i) mt[i] = 1812433253u * (mt[i - 1] ^ (mt[i - 1] >> 30)) + (uint32_t)i;
}

// Word k of the next block, from the state as it stands.  Applied to k = 0, 1, ... in place it is also the
// generator's one-word step T on a state whose oldest word sits at k.
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

// ---------------------------------------------------------------------------------------------- jump-ahead
// A polynomial over GF(2): bit k of word k / 64 is the coefficient of x^k.
using Poly = std::vector<uint64_t>;
constexpr int kPolyWords = (2 * kMtBits + 63) / 64 + 1;

inline bool poly_bit(const Poly &p, int64_t k) { return (p[k >> 6] >> (k & 63)) & 1u; }

// dst ^= src x^shift over src's lowest src_bits bits; terms past dst's end are dropped (callers keep them zero).
inline void poly_xor_shifted(Poly &dst, const Poly &src, int64_t shift, int64_t src_bits) {
    const int64_t w = shift >> 6, b = shift & 63, nd = (int64_t)dst.size();
    const int64_t nw = std::min<int64_t>((src_bits + 63) >> 6, (int64_t)src.size());
    for (int64_t k = 0; k < nw && k + w < nd; ++k) {
        const uint64_t v = src[k];
        if (!v) continue;
        dst[k + w] ^= v << b;
        if (b && k + w + 1 < nd) dst[k + w + 1] ^= v >> (64 - b);
    }
}

// phi by Berlekamp-Massey over the lowest output bit of init_genrand(5489)'s stream: 2 deg + 64 bits fix the
// minimal polynomial of the sequence, and MT19937's characteristic polynomial is irreducible, so that is phi.
// Returns an empty polynomial if the degree comes out other than 19937.
inline Poly mt_char_poly() {
    const int64_t N = 2 * kMtBits + 64;
    const int64_t NW = (N + 63) / 64 + 1;
    Poly rev(NW + 1, 0);   // bit N - 1 - t = output bit t, so s[t - L .. t] is one ascending window
    uint32_t st[kMtN];
    mt_init(st, 5489u);
    for (int64_t t = 0; t < N; ++t) {
        if (t % kMtN == 0) mt_twist(st);
        if (mt_temper(st[t % kMtN]) & 1u) rev[(N - 1 - t) >> 6] |= 1ull << ((N - 1 - t) & 63);
    }
    Poly C(NW + 1, 0), B(NW + 1, 0), T;
    C[0] = B[0] = 1;
    int64_t L = 0, m = 1;
    for (int64_t t = 0; t < N; ++t) {
        // d = sum_{i=0..L} C_i s[t - i] = parity(C & rev >> (N - 1 - t)) over L + 1 bits
        const int64_t o = N - 1 - t, ow = o >> 6, ob = o & 63;
        uint64_t acc = 0;
        for (int64_t k = 0; k <= (L >> 6); ++k) {
            uint64_t win = rev[ow + k] >> ob;
            if (ob && ow + k + 1 < (int64_t)rev.size()) win |= rev[ow + k + 1] << (64 - ob);
            if (k == (L >> 6) && ((L + 1) & 63)) win &= (1ull << ((L + 1) & 63)) - 1;
            acc ^= C[k] & win;
        }
        if (!(__builtin_popcountll(acc) & 1)) {
            ++m;
        } else if (2 * L <= t) {
            T = C;
            poly_xor_shifted(C, B, m, (int64_t)B.size() * 64 - m);
            L = t + 1 - L;
            B = T;
            m = 1;
        } else {
            poly_xor_shifted(C, B, m, (int64_t)B.size() * 64 - m);
            ++m;
        }
    }
    if (L != kMtBits) return Poly();
    Poly phi(kPolyWords, 0);   // the reciprocal of the connection polynomial: phi_{L - i} = C_i
    for (int64_t i = 0; i <= L; ++i)
        if (poly_bit(C, i)) phi[(L - i) >> 6] |= 1ull << ((L - i) & 63);
    return phi;
}

// p mod phi for p of degree < 2 deg(phi), in place.
inline void poly_reduce(Poly &p, const Poly &phi) {
    for (int64_t k = 2 * kMtBits - 2; k >= kMtBits; --k)
        if (poly_bit(p, k)) poly_xor_shifted(p, phi, k - kMtBits, kMtBits + 1);
}

inline Poly poly_square_mod(const Poly &p, const Poly &phi) {
    Poly q(kPolyWords, 0);
    for (int64_t k = 0; k < kMtBits; ++k)
        if (poly_bit(p, k)) q[(2 * k) >> 6] |= 1ull << ((2 * k) & 63);
    poly_reduce(q, phi);
    return q;
}

inline Poly poly_times_x_mod(const Poly &p, const Poly &phi) {
    Poly q(kPolyWords, 0);
    poly_xor_shifted(q, p, 1, kMtBits);
    poly_reduce(q, phi);
    return q;
}

// x^d mod phi by square-and-multiply (the multiplier is always x).
inline Poly poly_x_pow_mod(uint64_t d, const Poly &phi) {
    Poly p(kPolyWords, 0);
    p[0] = 1;
    for (int b = 63; b >= 0; --b) {
        p = poly_square_mod(p, phi);
        if ((d >> b) & 1) p = poly_times_x_mod(p, phi);
    }
    return p;
}

inline int poly_degree(const Poly &p) {
    for (int k = kMtBits - 1; k >= 0; --k)
        if (poly_bit(p, k)) return k;
    return -1;
}

// The state p(T) s on the host, s and the result at a block boundary (the next word is a block's word 0), as the
// device's jump kernel computes it.  p = x^d mod phi with d a multiple of 624.
inline void mt_jump(const uint32_t *s, const Poly &p, uint32_t *out) {
    uint32_t acc[kMtN] = {0};
    int idx = 0;
    for (int k = poly_degree(p); k >= 0; --k) {
        acc[idx] = mt_twist_word(acc, idx);
        idx = idx + 1 == kMtN ? 0 : idx + 1;
        if (poly_bit(p, k))
            for (int i = 0; i < kMtN; ++i) acc[(idx + i) % kMtN] ^= s[i];
    }
    for (int i = 0; i < kMtN; ++i) out[i] = acc[(idx + i) % kMtN];
}

}  // namespace mt
}  // namespace xrs

// local_rule.cuh -- the reference's local.py restated per cell, for one K-layer stack.  Everything here is
// __host__ __device__ and free of CUDA calls: the CPU tests compile this header with g++ (FMA contraction off, as
// the library) and reproduce every golden array of the unmodified reference with it.
//
// The reference turns each cell's K values into Python scalars (`.item()`): integer cells become int, float cells
// exact float, bool cells bool.  A `Val` is such a scalar.  What happens next depends on the function
// (DESIGN.md section 4.13):
//   cell_stats      np.<func>(tuple): the tuple becomes an array of one kind for the whole call (`ak`: bool when
//                   every layer is bool, float when any is float, else int64), then NumPy's reductions run;
//   positions, rank Python's own comparisons, exact between int and float;
//   frequencies     a NumPy scalar of the ref layer's type against the Python scalar (NEP 50);
//   popularity      np.array(tuple) (kind `ak`), a Counter, sorted distinct values.
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/xrs_b200.h"

#ifndef __CUDACC__
#define __host__
#define __device__
#endif

namespace xrs {
namespace lc {

enum Op { kSum = 0, kMean, kMedian, kMin, kMax, kStd, kLesser, kEqual, kGreater, kLowest, kHighest, kPopularity,
          kRank, kNumOps };
enum Kind { kFloat = 0, kInt = 1, kBool = 2 };

// per-call flags, OR-ed over the cells
constexpr unsigned kFlagNan = 1;          // some cell's result is NaN
constexpr unsigned kFlagIndexError = 2;   // rank / popularity: an index below -length (IndexError)
constexpr unsigned kFlagTypeError = 4;    // rank / popularity: a float ref reached the list index (TypeError)
constexpr unsigned kFlagFloatResult = 8;  // rank / popularity: some result is a float
constexpr unsigned kFlagIntResult = 16;   // rank / popularity: some result is an int that is not a bool

struct Val {
    double f;    // kind kFloat
    int64_t i;   // kInt, kBool (0 / 1)
    int kind;
};

__host__ __device__ inline Val fval(double f) { return Val{f, 0, kFloat}; }
__host__ __device__ inline Val ival(int64_t i, int kind) { return Val{0.0, i, kind}; }

// A cell of C++ type T as the Python scalar `.item()` gives (uint64 cells are below 2**63).
template <typename T> __host__ __device__ inline Val load(T x) {
    if constexpr (sizeof(T) == 1 && T(2) == T(1)) return ival(x ? 1 : 0, kBool);   // bool
    else if constexpr (T(0.5) != T(0)) return fval((double)x);
    else return ival((int64_t)x, kInt);
}

__host__ __device__ inline bool is_nan(const Val &v) { return v.kind == kFloat && v.f != v.f; }
__host__ __device__ inline double as_double(const Val &v) { return v.kind == kFloat ? v.f : (double)v.i; }

// The value in an array of kind ak (np.array(tuple)): ints and bools widen to float64 in a float array, bools
// to int64 in an int array.
__host__ __device__ inline Val as_array(const Val &v, int ak) {
    if (ak == kFloat) return fval(as_double(v));
    return ival(v.i, ak);
}

// Python's comparison of two scalars, exact between int and float: -1, 0 or 1 (no NaN).
__host__ __device__ inline int cmp_int_double(int64_t i, double d) {
    if (d >= 9223372036854775808.0) return -1;
    if (d < -9223372036854775808.0) return 1;
    const int64_t t = (int64_t)d;   // d truncated, exact in this range
    if (i != t) return i < t ? -1 : 1;
    const double frac = d - (double)t;
    return frac > 0 ? -1 : (frac < 0 ? 1 : 0);
}
__host__ __device__ inline int py_cmp(const Val &a, const Val &b) {
    if (a.kind != kFloat && b.kind != kFloat) return a.i < b.i ? -1 : (a.i > b.i ? 1 : 0);
    if (a.kind == kFloat && b.kind == kFloat) return a.f < b.f ? -1 : (a.f > b.f ? 1 : 0);
    if (a.kind == kFloat) return -cmp_int_double(b.i, a.f);
    return cmp_int_double(a.i, b.f);
}

// d rounded to float16 (to nearest, ties to even; beyond the largest half to +-inf).  The step is found from d's
// exponent bits, so the device code makes no library calls.
__host__ __device__ inline double round_f16(double d) {
    if (d != d) return d;
    const double a = fabs(d);
    if (a >= 65520.0) return copysign((double)INFINITY, d);
    union { double d; uint64_t u; } q, iq;   // the step and its inverse, powers of two
    q.d = 5.9604644775390625e-08;            // 2**-24, the subnormal step
    iq.d = 16777216.0;
    if (a >= 6.103515625e-05) {
        union { double d; uint64_t u; } b;
        b.d = a;
        q.u = ((b.u >> 52) - 10) << 52;      // 2**(e - 10) for a in [2**e, 2**(e+1)): 11 significant bits
        iq.u = (2056 - (b.u >> 52)) << 52;   // 2**(10 - e)
    }
    return copysign(rint(a * iq.d) * q.d, d);
}

// The ref layer's cell as the NumPy scalar the reference iterates: its value, the float width it compares in
// (0 for int and bool refs) and `ref - 1` computed in its own type.
struct Ref {
    Val v;
    int fbits;     // 16, 32, 64, or 0
    int64_t idx;   // ref - 1 wrapped in the ref's integer type (int64 for bool); INT64_MAX stands for 2**64 - 1
    double idxf;   // ref - 1 in the ref's float type
};

// code: the ref layer's xrs_dtype; f16: its cells are float16 carried as float32.
__host__ __device__ inline Ref make_ref(const Val &v, int code, bool f16) {
    Ref r{v, 0, 0, 0.0};
    const uint64_t u = (uint64_t)v.i - 1u;
    switch (code) {
        case XRS_F32:
            r.fbits = f16 ? 16 : 32;
            r.idxf = f16 ? round_f16(v.f - 1.0) : (double)((float)v.f - 1.0f);
            break;
        case XRS_F64: r.fbits = 64; r.idxf = v.f - 1.0; break;
        case XRS_I8: r.idx = (int8_t)(uint8_t)u; break;
        case XRS_I16: r.idx = (int16_t)(uint16_t)u; break;
        case XRS_I32: r.idx = (int32_t)(uint32_t)u; break;
        case XRS_U8: r.idx = (uint8_t)u; break;
        case XRS_U16: r.idx = (uint16_t)u; break;
        case XRS_U32: r.idx = (uint32_t)u; break;
        case XRS_U64: r.idx = v.i == 0 ? INT64_MAX : (int64_t)u; break;
        default: r.idx = (int64_t)u; break;   // int64 wraps; bool - 1 is an int64
    }
    return r;
}

__host__ __device__ inline int fcmp(double a, double b) { return a < b ? -1 : (a > b ? 1 : (a == b ? 0 : 2)); }

// The data value against the ref as NumPy compares them: -1 (data < ref), 0, 1, or 2 (unordered).  A float ref
// compares in its own type: the data value goes to float64 (a Python int through float64, as NumPy converts it),
// then rounds to the ref's width.  An int or bool ref compares in float64 against a float, exactly against an int.
__host__ __device__ inline int freq_cmp(const Ref &r, const Val &x) {
    if (r.fbits) {
        double d = as_double(x);
        if (r.fbits == 32) d = (double)(float)d;
        else if (r.fbits == 16) d = round_f16(d);
        return fcmp(d, r.v.f);
    }
    if (x.kind == kFloat) return fcmp(x.f, (double)r.v.i);
    return x.i < r.v.i ? -1 : (x.i > r.v.i ? 1 : 0);
}

// `list[ref - 1]` for a list of n items: 0 with *pos set, 1 when the index is >= n (the reference's NaN),
// kFlagIndexError below -n, kFlagTypeError for a float ref that gets this far.
__host__ __device__ inline unsigned list_index(const Ref &r, int64_t n, int64_t *pos) {
    if (r.fbits) return r.idxf >= (double)n ? 1u : kFlagTypeError;
    if (r.idx >= n) return 1u;
    if (r.idx < -n) return kFlagIndexError;
    *pos = r.idx < 0 ? r.idx + n : r.idx;
    return 0u;
}

// ---------------------------------------------------------------------------------------------- NumPy reductions
// NumPy's pairwise sum of x(lo) .. x(lo + n - 1), n <= 128: sequential from +0.0 below 8 items, else eight strided
// accumulators combined as ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the tail.
template <class X> __host__ __device__ inline double pw_block(const X &x, int64_t lo, int64_t n) {
    if (n < 8) {
        double s = 0.0;
        for (int64_t j = 0; j < n; ++j) s += x(lo + j);
        return s;
    }
    double r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = x(lo + j);
    int64_t i = 8;
    for (; i < n - n % 8; i += 8) {
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] += x(lo + i + j);
    }
    double s = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (; i < n; ++i) s += x(lo + i);
    return s;
}

__host__ __device__ inline int64_t pw_split(int64_t n) { return n / 2 - (n / 2) % 8; }

// Above 128 items NumPy splits at m = n/2 - (n/2) % 8 and adds the halves' sums: the same tree, walked with an
// explicit stack.
template <class X> __host__ __device__ inline double pw_large(const X &x, int64_t n) {
    int64_t lo_[64], n_[64];
    double left[64];
    bool right[64];
    int sp = 0;
    lo_[0] = 0;
    n_[0] = n;
    right[0] = false;
    for (;;) {
        if (n_[sp] > 128) {   // descend into the left half
            const int64_t m = pw_split(n_[sp]);
            lo_[sp + 1] = lo_[sp];
            n_[sp + 1] = m;
            right[sp + 1] = false;
            ++sp;
            continue;
        }
        double s = pw_block(x, lo_[sp], n_[sp]);
        while (sp > 0 && right[sp]) {   // a right half completes its parent
            --sp;
            s = left[sp] + s;
        }
        if (sp == 0) return s;
        left[sp - 1] = s;               // a left half: the parent's right half is next
        const int64_t m = n_[sp];
        lo_[sp] = lo_[sp - 1] + m;
        n_[sp] = n_[sp - 1] - m;
        right[sp] = true;
    }
}

// np.sum in float64: the pairwise sum added to the +0.0 identity
template <class X> __host__ __device__ inline double np_sum(const X &x, int64_t n) {
    return (n <= 128 ? pw_block(x, 0, n) : pw_large(x, n)) + 0.0;
}

// np.max (least: np.min) of n NaN-free doubles, including which of equal +-0.0 comes out.  NumPy's contiguous
// reduction keeps x(0) as its accumulator, folds whole 8-lane vectors of the rest lane by lane, reduces the lanes
// as upper half against lower half, and folds the tail one item at a time; every step keeps its second operand
// unless the first is strictly larger (smaller).  Pinned by the goldens.
template <class X> __host__ __device__ inline double np_extreme(const X &x, int64_t n, bool least) {
    auto pick = [least](double a, double b) { return (least ? a < b : a > b) ? a : b; };
    const double x0 = x(0);
    const int64_t nvec = (n - 1) / 8;
    double r = x0;
    if (nvec > 0) {
        double v[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            double l = x0;
            for (int64_t t = 0; t < nvec; ++t) l = pick(l, x(1 + i + 8 * t));
            v[i] = l;
        }
        double t3[4], t6[2];
#pragma unroll
        for (int i = 0; i < 4; ++i) t3[i] = pick(v[i + 4], v[i]);
#pragma unroll
        for (int i = 0; i < 2; ++i) t6[i] = pick(t3[i + 2], t3[i]);
        r = pick(t6[0], t6[1]);
    }
    for (int64_t j = 1 + 8 * nvec; j < n; ++j) r = pick(r, x(j));
    return r;
}

// ---------------------------------------------------------------------------------------------- the rule
struct Result {
    int64_t bits;    // an int64, or a double's bits when kind == kFloat
    int kind;        // kFloat, kInt, kBool
    unsigned flags;  // kFlag* of this cell
};

__host__ __device__ inline Result res_double(double d) {
    Result r;
    union { double d; int64_t i; } u;
    u.d = d;
    r.bits = u.i;
    r.kind = kFloat;
    r.flags = d != d ? kFlagNan : 0u;
    return r;
}
__host__ __device__ inline Result res_int(int64_t i, int kind) { return Result{i, kind, 0u}; }
__host__ __device__ inline Result res_nan() { return res_double(NAN); }
// counts, positions and combine ids: -1 marks NaN
__host__ __device__ inline Result res_count_nan() { return Result{-1, kInt, kFlagNan}; }
// rank / popularity results are typed per cell
__host__ __device__ inline Result res_elem(const Val &v) {
    if (v.kind == kFloat) {
        Result r = res_double(v.f);
        r.flags |= kFlagFloatResult;
        return r;
    }
    return Result{v.i, v.kind, v.kind == kInt ? kFlagIntResult : 0u};
}

// k-th smallest (0-based) of n NaN-free doubles
template <class Y> __host__ __device__ inline double kth_smallest(const Y &y, int64_t n, int64_t k) {
    for (int64_t i = 0; i < n; ++i) {
        const double yi = y(i);
        int64_t lt = 0, le = 0;
        for (int64_t j = 0; j < n; ++j) {
            const double yj = y(j);
            lt += yj < yi;
            le += yj <= yi;
        }
        if (lt <= k && k < le) return yi;
    }
    return NAN;   // not reached
}

// The result of `op` for one cell.  x(j) is layer j's value (a Val), ak the stack's array kind, ref the cell's ref
// value (frequencies, rank, popularity).
template <class X>
__host__ __device__ inline Result cell(int op, int64_t K, int ak, const X &x, const Ref &ref) {
    // NaN cells: sums propagate NaN by themselves; the single-pass functions note a NaN as they read (xn, xdn);
    // the order statistics check first
    bool nan = false;
    auto xd = [&](int64_t j) { return as_double(x(j)); };
    auto xn = [&](int64_t j) {
        const Val v = x(j);
        nan |= is_nan(v);
        return v;
    };
    auto xdn = [&](int64_t j) {
        const double d = xd(j);
        nan |= d != d;
        return d;
    };
    auto any_nan = [&]() {
        for (int64_t j = 0; j < K; ++j)
            if (is_nan(x(j))) return true;
        return false;
    };
    switch (op) {
        case kSum:
            if (ak == kFloat) return res_double(np_sum(xd, K));
            else {
                uint64_t s = 0;
                for (int64_t j = 0; j < K; ++j) s += (uint64_t)x(j).i;
                return res_int((int64_t)s, kInt);
            }
        case kMin:
        case kMax:
            if (ak == kFloat) {
                const double m = np_extreme(xdn, K, op == kMin);
                return nan ? res_nan() : res_double(m);
            } else {
                int64_t m = x(0).i;
                for (int64_t j = 1; j < K; ++j) {
                    const int64_t v = x(j).i;
                    m = op == kMin ? (v < m ? v : m) : (v > m ? v : m);
                }
                return res_int(m, ak);
            }
        case kMean: return res_double(np_sum(xd, K) / (double)K);
        case kStd: {
            const double m = np_sum(xd, K) / (double)K;
            auto sq = [&](int64_t j) {
                const double d = xd(j) - m;
                return d * d;
            };
            return res_double(sqrt(np_sum(sq, K) / (double)K));
        }
        case kMedian: {
            if (any_nan()) return res_nan();
            const double lo = kth_smallest(xd, K, (K - 1) / 2);
            if (K % 2) return res_double((0.0 + lo) / 1.0);
            const double hi = kth_smallest(xd, K, K / 2);
            return res_double((0.0 + lo + hi) / 2.0);
        }
        case kLesser:
        case kEqual:
        case kGreater: {
            const int want = op == kLesser ? -1 : (op == kEqual ? 0 : 1);
            int64_t c = 0;
            for (int64_t j = 0; j < K; ++j) c += freq_cmp(ref, xn(j)) == want;
            return nan ? res_count_nan() : res_int(c, kInt);
        }
        case kLowest:
        case kHighest: {
            const int better = op == kLowest ? -1 : 1;
            int64_t b = 0;
            Val bv = xn(0);
            for (int64_t j = 1; j < K; ++j) {
                const Val v = xn(j);
                if (py_cmp(v, bv) == better) {
                    b = j;
                    bv = v;
                }
            }
            return nan ? res_count_nan() : res_int(b + 1, kInt);
        }
        case kRank: {
            if (any_nan()) return res_nan();
            int64_t p = 0;
            const unsigned e = list_index(ref, K, &p);
            if (e == 1u) return res_nan();
            if (e) return Result{0, kInt, e};
            // the item at position p of the stable sort
            for (int64_t i = 0; i < K; ++i) {
                const Val vi = x(i);
                int64_t pos = 0;
                for (int64_t j = 0; j < K; ++j) {
                    const int c = py_cmp(x(j), vi);
                    pos += c < 0 || (c == 0 && j < i);
                }
                if (pos == p) return res_elem(vi);
            }
            return res_nan();   // not reached
        }
        case kPopularity: {
            if (any_nan()) return res_nan();
            auto y = [&](int64_t j) { return as_array(x(j), ak); };
            auto first = [&](int64_t i) {   // y(i) is the first occurrence of its value (+-0.0 are one value)
                const Val yi = y(i);
                for (int64_t j = 0; j < i; ++j)
                    if (py_cmp(y(j), yi) == 0) return false;
                return true;
            };
            int64_t D = 0;
            for (int64_t i = 0; i < K; ++i) D += first(i);
            if (D >= K) return res_nan();
            if (D == 1) return res_elem(y(0));
            int64_t p = 0;
            const unsigned e = list_index(ref, D, &p);
            if (e == 1u) return res_nan();
            if (e) return Result{0, kInt, e};
            // walk up the distinct values from the least, p steps, each an O(K) scan for the least value above the
            // current one; taking only strictly smaller candidates keeps each value's first occurrence
            int64_t cur = 0;
            for (int64_t j = 1; j < K; ++j)
                if (py_cmp(y(j), y(cur)) < 0) cur = j;
            for (int64_t step = 0; step < p; ++step) {
                const Val c = y(cur);
                int64_t next = -1;
                for (int64_t j = 0; j < K; ++j) {
                    const Val v = y(j);
                    if (py_cmp(v, c) > 0 && (next < 0 || py_cmp(v, y(next)) < 0)) next = j;
                }
                cur = next;
            }
            return res_elem(y(cur));
        }
    }
    return res_nan();
}

// ---------------------------------------------------------------------------------------------- combine
// Hash and equality of a cell's K-tuple as Python tuples compare: +-0.0 are one value (NaN cells never get here).
__host__ __device__ inline uint64_t mix64(uint64_t z) {
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}
__host__ __device__ inline uint64_t key_bits(const Val &v) {
    if (v.kind != kFloat) return (uint64_t)v.i;
    union { double d; uint64_t u; } c;
    c.d = v.f == 0.0 ? 0.0 : v.f;
    return c.u;
}
template <class X> __host__ __device__ inline uint64_t tuple_hash(int64_t K, const X &x) {
    uint64_t h = 0x9e3779b97f4a7c15ull;
    for (int64_t j = 0; j < K; ++j) h = mix64(h ^ key_bits(x(j)));
    return h;
}
template <class X, class Y> __host__ __device__ inline bool tuple_equal(int64_t K, const X &a, const Y &b) {
    for (int64_t j = 0; j < K; ++j)
        if (py_cmp(a(j), b(j)) != 0) return false;
    return true;
}

}  // namespace lc
}  // namespace xrs

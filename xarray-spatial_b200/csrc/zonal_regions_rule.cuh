// zonal_regions_rule.cuh -- zonal.regions (zonal.py:1406-1549 of the reference) restated per cell, so the
// labelling can run as a union-find.  Everything here is __host__ __device__ and free of CUDA calls: the CPU tests
// compile this header with g++ (FMA contraction off, as the library) and label rasters with a host union-find.
//
// The reference scans the raster twice in row-major order.  Its labels are fixed by three things (DESIGN.md
// section 4.12):
//   new uid   a non-NaN cell C gets a fresh uid iff no slot of its window that lies before C in row-major order
//             matches C; its uid is the number of such cells at or before it.
//   edges     (a) a cell that is not new joins its first earlier matching slot, in slot order;
//             (b) all matching slots of a non-NaN C join each other (C itself only when clamping puts it in its own
//             window).  Such an edge can join cells two apart.
//   label     the uid of the lowest-index cell of C's component, which is always a new-uid cell.
// A slot S matches C when close(data[S], data[C]); NaN never matches.
#pragma once
#include <stdint.h>

#include <type_traits>

#ifndef __CUDACC__
#define __host__
#define __device__
#endif

namespace xrs {
namespace zr {

constexpr uint32_t kNew = 1u << 8;   // code bit: the cell takes a fresh uid
constexpr uint32_t kNan = 1u << 9;   // code bit: the cell is NaN (no edges, NaN label)

// Slot s of the n-cell window as a row / column step, in the reference's order (zonal.py:1424-1452):
// n = 4: left, up, down, right; n = 8: the left column top to bottom, up, down, the right column top to bottom.
__host__ __device__ inline void slot_step(int n, int s, int &dr, int &dc) {
    if (n == 8) {
        dc = s < 3 ? -1 : (s < 5 ? 0 : 1);
        dr = s < 3 ? s - 1 : (s < 5 ? (s == 3 ? -1 : 1) : s - 6);
    } else {
        dr = s == 1 ? -1 : (s == 2 ? 1 : 0);
        dc = s == 0 ? -1 : (s == 3 ? 1 : 0);
    }
}

// Row-major index of slot s of cell (y, x), its row and column clamped to the raster.
__host__ __device__ inline int64_t slot_index(int n, int s, int64_t H, int64_t W, int64_t y, int64_t x) {
    int dr, dc;
    slot_step(n, s, dr, dc);
    int64_t r = y + dr, c = x + dc;
    r = r < 0 ? 0 : (r > H - 1 ? H - 1 : r);
    c = c < 0 ? 0 : (c > W - 1 ? W - 1 : c);
    return r * W + c;
}

template <typename T> __host__ __device__ inline bool is_nan(T v) {
    if constexpr (std::is_floating_point_v<T>) return v != v;
    else return false;
}

// |v - c| <= 1e-08 + 1e-05 |c| as numba evaluates it for the raster's type: floats subtract in their own type;
// signed integers subtract in int64 (wrapping for int64) and take |c| in their own type (so |int8 -128| is -128);
// unsigned integers subtract in uint64, wrapping.  Both sides are compared in float64.
template <typename T> __host__ __device__ inline bool close(T v, T c) {
    if constexpr (std::is_floating_point_v<T>) {
        T d = v - c;
        d = d < 0 ? -d : d;
        const T ac = c < 0 ? -c : c;
        return (double)d <= 1e-08 + 1e-05 * (double)ac;
    } else if constexpr (std::is_signed_v<T>) {
        const uint64_t u = (uint64_t)(int64_t)v - (uint64_t)(int64_t)c;
        const int64_t d = (int64_t)u < 0 ? (int64_t)(0 - u) : (int64_t)u;
        const T ac = c < 0 ? (T)(0 - (uint64_t)(int64_t)c) : c;
        return (double)d <= 1e-08 + 1e-05 * (double)ac;
    } else {
        const uint64_t d = (uint64_t)v - (uint64_t)c;
        return (double)d <= 1e-08 + 1e-05 * (double)c;
    }
}

// The code of cell (y, x): bit s set when slot s matches, kNew when no earlier slot matches, kNan for a NaN cell.
// get(r, c) returns the raster's cell.
template <typename T, typename Get>
__host__ __device__ inline uint32_t cell_code(int n, int64_t H, int64_t W, int64_t y, int64_t x, const Get &get) {
    const T c = get(y, x);
    if (is_nan(c)) return kNan;
    const int64_t k = y * W + x;
    uint32_t m = kNew;
    for (int s = 0; s < n; ++s) {
        const int64_t p = slot_index(n, s, H, W, y, x);
        if (close<T>(get(p / W, p % W), c)) {
            m |= 1u << s;
            if (p < k) m &= ~kNew;
        }
    }
    return m;
}

// Calls f(a, b) for the union edges cell (y, x) with `code` contributes: its matching slots joined to the first of
// them, and, unless it is new, the cell joined to its first earlier matching slot.
template <typename F>
__host__ __device__ inline void for_each_edge(int n, int64_t H, int64_t W, int64_t y, int64_t x, uint32_t code,
                                              const F &f) {
    if (code & kNan) return;
    const int64_t k = y * W + x;
    int64_t first = -1, adopt = -1;
    for (int s = 0; s < n; ++s) {
        if (!((code >> s) & 1u)) continue;
        const int64_t p = slot_index(n, s, H, W, y, x);
        if (first < 0) first = p;
        else if (p != first) f(first, p);
        if (adopt < 0 && p < k) adopt = p;
    }
    if (!(code & kNew)) f(k, adopt);
}

}  // namespace zr
}  // namespace xrs

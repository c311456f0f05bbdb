// zonal_hash.cu -- single-pass zonal.stats partials without knowing the zone ids in advance.
//
// zonal.py:280-332 discovers the ids with np.unique and sorts the raster by zone (argsort).
// Here the ids are discovered BY the streaming pass itself: a group-by aggregation into an
// open-addressing hash table keyed by the zone id.
//   * every thread streams quads of 4 consecutive cells (128-bit loads, UNROLL quads in flight
//     before any is consumed) and keeps a private accumulator for the run of equal zone ids it
//     is in (count, sum and sum of squares about a global pivot in f64, min / max);
//   * when the id changes the run is merged into a per-CTA shared-memory hash table
//     (atomicCAS on the key, native shared-memory atomics on the accumulators);
//   * at the end each CTA merges its table into the global table (same probing, global
//     atomics).  Tables from several GPUs are merged by key on the host (a few KB).
// 8 algorithmic bytes per cell (f32 values + i32 zones): HBM-bound.
#include <math.h>

#include <algorithm>

#include "common.cuh"

namespace xrs {

constexpr int kZhThreads = 256;
constexpr int kZhLocalCap = 1024;       // per-CTA table slots of the pair kernel (x2) and of float64 values
constexpr int kZhUnroll = 4;            // rows per lane in flight
constexpr int kZhSegRows = 256;         // rows per task
constexpr long long kZhEmpty = (long long)0x8000000000000000ULL;

struct ZhArgs {
    const void *values;
    const void *zones;
    int64_t n;
    int64_t W;      // row length of the raster (n = H * W); walking DOWN columns keeps runs long
    double pivot;
    const double *pivot_ptr;   // when not NULL the pivot is read from device memory (xrs_zonal_hash_run)
    const double *zone_pivots; // when not NULL: one pivot per slot of the (already populated) global table --
                               // the second pass, sums about the zones' own means
    int has_nodata;
    double nodata;
    long long *keys;
    unsigned long long *count;
    double *s1, *s2, *vmin, *vmax;
    int cap;  // global slots, power of two
    int *overflow;
    int *sentinel;  // when not NULL: set to 1 if an int64 zone equals the empty key (INT64_MIN), which the table
                    // cannot hold -- the host computes that one zone on its own
};

__device__ __forceinline__ unsigned zh_hash(long long key) {
    return (unsigned)(((unsigned long long)key * 0x9E3779B97F4A7C15ULL) >> 32);
}
__device__ __forceinline__ void zh_atomic_min(double *addr, double v) {
    unsigned long long *a = reinterpret_cast<unsigned long long *>(addr);
    unsigned long long old = *a;
    while (v < __longlong_as_double((long long)old)) {
        const unsigned long long assumed = old;
        old = atomicCAS(a, assumed, (unsigned long long)__double_as_longlong(v));
        if (old == assumed) break;
    }
}
__device__ __forceinline__ void zh_atomic_max(double *addr, double v) {
    unsigned long long *a = reinterpret_cast<unsigned long long *>(addr);
    unsigned long long old = *a;
    while (v > __longlong_as_double((long long)old)) {
        const unsigned long long assumed = old;
        old = atomicCAS(a, assumed, (unsigned long long)__double_as_longlong(v));
        if (old == assumed) break;
    }
}

// float32 values keep their per-CTA min / max as order-preserving int32 keys, so that the table
// update is one native ATOMS.MIN / ATOMS.MAX (shared memory has native atomics for 32-bit
// integers only: float and every 64-bit type compile to compare-and-swap loops) and a slot takes
// 36 bytes.  That buys 1408 slots per CTA inside the same 164 KB shared-memory carve-out as before
// (3 CTAs / SM; a larger carve-out leaves too little L1 for the loads in flight -- 2048 slots
// measured 20 % slower on coherent zones): a CTA that meets ~1000 distinct zones (scattered zone
// ids, the worst case of SURVEY.md 8d) no longer fills its table and falls back to global atomics.
__device__ __forceinline__ int zh_fkey(float f) {
    const int b = __float_as_int(f);
    return b ^ ((b >> 31) & 0x7fffffff);
}
__device__ __forceinline__ float zh_funkey(int k) { return __int_as_float(k ^ ((k >> 31) & 0x7fffffff)); }
template <typename VT> struct ZhMinMax { using type = double; };
template <> struct ZhMinMax<float> { using type = int; };
template <typename VT> struct ZhTable {
    static constexpr int kCap = sizeof(VT) == 4 ? 1408 : kZhLocalCap;   // need not be a power of two
    static constexpr size_t kBytes = (size_t)kCap * (8 + 8 + 8 + 2 * sizeof(typename ZhMinMax<VT>::type) + 4);
};

// find-or-insert in a per-CTA table of any size: start slot by multiply-shift range reduction
__device__ __forceinline__ int zh_slot_local(long long *keys, int cap, long long key, int max_probe) {
    unsigned s = __umulhi(zh_hash(key), (unsigned)cap);
    for (int p = 0; p < max_probe; ++p) {
        const long long k = keys[s];
        if (k == key) return (int)s;
        if (k == kZhEmpty) {
            const long long prev = (long long)atomicCAS(reinterpret_cast<unsigned long long *>(&keys[s]),
                                                        (unsigned long long)kZhEmpty, (unsigned long long)key);
            if (prev == kZhEmpty || prev == key) return (int)s;
        }
        s = (s + 1 == (unsigned)cap) ? 0u : s + 1;
    }
    return -1;
}

// find-or-insert `key`; returns the slot or -1 when `max_probe` slots were all taken by others
__device__ __forceinline__ int zh_slot(long long *keys, int cap, long long key, int max_probe) {
    unsigned s = zh_hash(key) & (unsigned)(cap - 1);
    for (int p = 0; p < max_probe; ++p) {
        const long long k = keys[s];
        if (k == key) return (int)s;
        if (k == kZhEmpty) {
            const long long prev = (long long)atomicCAS(reinterpret_cast<unsigned long long *>(&keys[s]),
                                                        (unsigned long long)kZhEmpty, (unsigned long long)key);
            if (prev == kZhEmpty || prev == key) return (int)s;
        }
        s = (s + 1) & (unsigned)(cap - 1);
    }
    return -1;
}

// read-only lookup in a populated table; -1 when the key is absent
__device__ __forceinline__ int zh_find(const long long *keys, int cap, long long key) {
    unsigned s = zh_hash(key) & (unsigned)(cap - 1);
    for (int p = 0; p < cap; ++p) {
        const long long k = keys[s];
        if (k == key) return (int)s;
        if (k == kZhEmpty) return -1;
        s = (s + 1) & (unsigned)(cap - 1);
    }
    return -1;
}

template <typename ZT> __device__ __forceinline__ bool zh_key(ZT z, long long &key) {
    if constexpr (sizeof(ZT) == 4 && ZT(0.5) == ZT(0)) {  // int32
        key = (long long)z;
        return true;
    } else if constexpr (sizeof(ZT) == 8 && ZT(0.5) == ZT(0)) {  // int64
        key = (long long)z;
        return key != kZhEmpty;
    } else {  // float / double zones: finite values only (zonal.py:290), -0.0 folded into +0.0
        const double d = (double)z + 0.0;
        if (!(fabs(d) <= 1.7976931348623157e308)) return false;
        key = __double_as_longlong(d);
        return true;
    }
}

struct ZhRun {
    double s1, s2;
    float mnf, mxf;     // used for float values
    double mnd, mxd;    // used for double values
    unsigned cnt;
};

template <typename VT> __device__ __forceinline__ void zh_reset(ZhRun &r) {
    r.s1 = r.s2 = 0.0;
    r.cnt = 0u;
    r.mnf = INFINITY; r.mxf = -INFINITY;
    r.mnd = INFINITY; r.mxd = -INFINITY;
}

// finite and != nodata (zonal.py:159).  The nodata comparison happens in the values' dtype, like
// NumPy's `zone_values != nodata_values` with a Python scalar.
template <typename VT> __device__ __forceinline__ bool zh_valid(VT v, const ZhArgs &a) {
    if constexpr (sizeof(VT) == 4) return (fabsf(v) <= 3.402823466e38f) && !(a.has_nodata && v == (float)a.nodata);
    else return (fabs(v) <= 1.7976931348623157e308) && !(a.has_nodata && v == a.nodata);
}

template <typename VT> __device__ __forceinline__ void zh_add(ZhRun &r, VT v, const ZhArgs &a, double pivot) {
    if (zh_valid<VT>(v, a)) {
        const double d = (double)v - pivot;
        r.s1 += d;
        r.s2 = fma(d, d, r.s2);
        if constexpr (sizeof(VT) == 4) {
            r.mnf = fminf(r.mnf, v);
            r.mxf = fmaxf(r.mxf, v);
        } else {
            r.mnd = fmin(r.mnd, v);
            r.mxd = fmax(r.mxd, v);
        }
        r.cnt += 1u;
    }
}

// four cells of one zone at once, branch-free, with short dependency chains (tree sums)
template <typename VT> __device__ __forceinline__ void zh_add4(ZhRun &r, const VT (&v)[4], const ZhArgs &a, double pivot) {
    bool ok[4];
    double d[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        ok[k] = zh_valid<VT>(v[k], a);
        d[k] = ok[k] ? (double)v[k] - pivot : 0.0;
    }
    r.s1 += (d[0] + d[1]) + (d[2] + d[3]);
    r.s2 += fma(d[0], d[0], d[1] * d[1]) + fma(d[2], d[2], d[3] * d[3]);
    r.cnt += (unsigned)ok[0] + (unsigned)ok[1] + (unsigned)ok[2] + (unsigned)ok[3];
    if constexpr (sizeof(VT) == 4) {
        const float inf = INFINITY;
        r.mnf = fminf(r.mnf, fminf(fminf(ok[0] ? v[0] : inf, ok[1] ? v[1] : inf), fminf(ok[2] ? v[2] : inf, ok[3] ? v[3] : inf)));
        r.mxf = fmaxf(r.mxf, fmaxf(fmaxf(ok[0] ? v[0] : -inf, ok[1] ? v[1] : -inf), fmaxf(ok[2] ? v[2] : -inf, ok[3] ? v[3] : -inf)));
    } else {
        const double inf = INFINITY;
        r.mnd = fmin(r.mnd, fmin(fmin(ok[0] ? v[0] : inf, ok[1] ? v[1] : inf), fmin(ok[2] ? v[2] : inf, ok[3] ? v[3] : inf)));
        r.mxd = fmax(r.mxd, fmax(fmax(ok[0] ? v[0] : -inf, ok[1] ? v[1] : -inf), fmax(ok[2] ? v[2] : -inf, ok[3] ? v[3] : -inf)));
    }
}

template <typename T> struct ZhQuad { T v[4]; };
template <typename T> __device__ __forceinline__ ZhQuad<T> zh_load(const T *p, int64_t i, int64_t n, bool al) {
    ZhQuad<T> q;
    if (al && i + 4 <= n) {
        if constexpr (sizeof(T) == 4) {
            const int4 r = __ldcs(reinterpret_cast<const int4 *>(p + i));
            memcpy(&q.v[0], &r, 16);
        } else {
            const int4 r0 = __ldcs(reinterpret_cast<const int4 *>(p + i));
            const int4 r1 = __ldcs(reinterpret_cast<const int4 *>(p + i + 2));
            memcpy(&q.v[0], &r0, 16);
            memcpy(&q.v[2], &r1, 16);
        }
    } else {
#pragma unroll
        for (int k = 0; k < 4; ++k) q.v[k] = (i + k < n) ? p[i + k] : T(0);
    }
    return q;
}

// ZP: sums about per-zone pivots (a.zone_pivots; the second pass) instead of the one global pivot
template <typename VT, typename ZT, bool ZP>
__global__ void __launch_bounds__(kZhThreads, 3) zonal_hash_kernel(const __grid_constant__ ZhArgs a_in) {
    ZhArgs a = a_in;
    if (a.pivot_ptr != nullptr) a.pivot = *a.pivot_ptr;
    using MM = typename ZhMinMax<VT>::type;
    constexpr int kCap = ZhTable<VT>::kCap;
    extern __shared__ __align__(16) unsigned char zh_smem[];
    long long *s_keys = reinterpret_cast<long long *>(zh_smem);
    double *s_s1 = reinterpret_cast<double *>(s_keys + kCap);
    double *s_s2 = s_s1 + kCap;
    MM *s_mn = reinterpret_cast<MM *>(s_s2 + kCap);
    MM *s_mx = s_mn + kCap;
    unsigned *s_cnt = reinterpret_cast<unsigned *>(s_mx + kCap);
    for (int i = threadIdx.x; i < kCap; i += blockDim.x) {
        s_keys[i] = kZhEmpty;
        s_s1[i] = 0.0; s_s2[i] = 0.0; s_cnt[i] = 0u;
        if constexpr (sizeof(VT) == 4) { s_mn[i] = zh_fkey(INFINITY); s_mx[i] = zh_fkey(-INFINITY); }
        else { s_mn[i] = INFINITY; s_mx[i] = -INFINITY; }
    }
    __syncthreads();

    const VT *values = reinterpret_cast<const VT *>(a.values);
    const ZT *zones = reinterpret_cast<const ZT *>(a.zones);
    const bool v_al = (reinterpret_cast<uintptr_t>(values) & 15) == 0;
    const bool z_al = (reinterpret_cast<uintptr_t>(zones) & 15) == 0;

    ZhRun run;
    zh_reset<VT>(run);
    ZT cur_z = ZT(0);
    bool have = false, cur_ok = false;
    long long cur_key = 0;
    double cur_p = a.pivot;   // the shift of the lane's current run: global, or (ZP) its zone's

    // merge (key, cnt, s1, s2, mn, mx) into the CTA table, spilling to the global table when the
    // CTA sees more distinct zones than its table holds
    auto merge = [&](long long key, unsigned cnt, double s1, double s2, double mn, double mx) {
        int s = zh_slot_local(s_keys, kCap, key, 48);
        if (s >= 0) {
            if (cnt) {
                atomicAdd(&s_cnt[s], cnt);
                atomicAdd(&s_s1[s], s1);
                atomicAdd(&s_s2[s], s2);
                if constexpr (sizeof(VT) == 4) {
                    atomicMin(&s_mn[s], zh_fkey((float)mn));   // mn / mx came from float32 cells: exact
                    atomicMax(&s_mx[s], zh_fkey((float)mx));
                } else {
                    zh_atomic_min(&s_mn[s], mn);
                    zh_atomic_max(&s_mx[s], mx);
                }
            }
        } else {
            s = zh_slot(a.keys, a.cap, key, a.cap);
            if (s < 0) { *a.overflow = 1; }
            else if (cnt) {
                atomicAdd(&a.count[s], (unsigned long long)cnt);
                atomicAdd(&a.s1[s], s1);
                atomicAdd(&a.s2[s], s2);
                zh_atomic_min(&a.vmin[s], mn);
                zh_atomic_max(&a.vmax[s], mx);
            }
        }
    };
    // Flush the private run.  Called by ALL 32 lanes together (`need` says which lanes really
    // have something to flush).  Zone boundaries usually hit a whole warp-row at once, with every
    // lane leaving the same zone: then the 32 runs are first combined with warp shuffles and
    // lane 0 alone touches the table, instead of 32 lanes serialising on the same five atomics.
    // A zone is registered even when its run holds no valid value (count 0): zones without valid
    // cells must still be reported (NaN row, zonal.py:153-162).
    auto flush_all = [&](bool need) {
        const unsigned full = 0xffffffffu;
        need = need && cur_ok;
        const long long key0 = __shfl_sync(full, cur_key, 0);
        const bool uniform = __all_sync(full, need && cur_key == key0);
        double mn = sizeof(VT) == 4 ? (double)run.mnf : run.mnd;
        double mx = sizeof(VT) == 4 ? (double)run.mxf : run.mxd;
        if (uniform) {
            unsigned cnt = __reduce_add_sync(full, run.cnt);
            double s1 = run.s1, s2 = run.s2;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                s1 += __shfl_xor_sync(full, s1, o);
                s2 += __shfl_xor_sync(full, s2, o);
                mn = fmin(mn, __shfl_xor_sync(full, mn, o));
                mx = fmax(mx, __shfl_xor_sync(full, mx, o));
            }
            if ((threadIdx.x & 31) == 0) merge(key0, cnt, s1, s2, mn, mx);
        } else if (need) {
            merge(cur_key, run.cnt, run.s1, run.s2, mn, mx);
        }
        __syncwarp();
        if (need) zh_reset<VT>(run);
    };

    // Traversal: the raster is cut into strips of 128 columns x segments of kZhSegRows rows; a
    // warp owns a (segment, strip) task and walks down its rows, lane l owning columns
    // 4l .. 4l+3 (one 128-bit load per array per row, 512 contiguous bytes per warp-row).
    // Zone rasters are spatially coherent, so a lane's run of equal zone ids lasts for many
    // rows and the private accumulator is flushed rarely.  All 32 lanes execute every
    // iteration (lanes past the raster's right edge just see nv = 0), so the warp stays
    // converged and can use warp collectives.
    const int lane = threadIdx.x & 31;
    const int64_t H = a.n / a.W;
    const int64_t n_strips = (a.W + 127) / 128;
    const int64_t n_segs = (H + kZhSegRows - 1) / kZhSegRows;
    const int64_t n_tasks = n_strips * n_segs;
    const int64_t warps_total = (int64_t)gridDim.x * (kZhThreads / 32);
    const bool row_vec = v_al && z_al && (a.W % 4 == 0);
    for (int64_t task = (int64_t)blockIdx.x * (kZhThreads / 32) + (threadIdx.x >> 5); task < n_tasks;
         task += warps_total) {
        const int64_t seg = task / n_strips, strip = task % n_strips;
        const int64_t x = strip * 128 + 4 * lane;
        const int64_t y0 = seg * kZhSegRows, y1 = min(y0 + (int64_t)kZhSegRows, H);
        const int nv = (int)max((int64_t)0, min((int64_t)4, a.W - x));
        // whole strip inside the raster, 16-byte aligned rows: plain 128-bit loads, no bounds logic
        const bool strip_fast = row_vec && (strip * 128 + 128 <= a.W);
        const VT *vrow = values + y0 * a.W + x;
        const ZT *zrow = zones + y0 * a.W + x;
        for (int64_t y = y0; y < y1; y += kZhUnroll, vrow += kZhUnroll * a.W, zrow += kZhUnroll * a.W) {
            ZhQuad<VT> v[kZhUnroll];
            ZhQuad<ZT> z[kZhUnroll];
            const bool batch_fast = strip_fast && (y + kZhUnroll <= y1);
            if (batch_fast) {
#pragma unroll
                for (int u = 0; u < kZhUnroll; ++u) {
                    v[u] = zh_load<VT>(vrow + u * a.W, 0, 4, true);
                    z[u] = zh_load<ZT>(zrow + u * a.W, 0, 4, true);
                }
            } else {
#pragma unroll
                for (int u = 0; u < kZhUnroll; ++u) {
                    const int nvu = (y + u < y1) ? nv : 0;
                    v[u] = zh_load<VT>(vrow + u * a.W, 0, nvu, row_vec);
                    z[u] = zh_load<ZT>(zrow + u * a.W, 0, nvu, row_vec);
                }
            }
            // ---- the whole batch inside the lanes' current zones: one vote per 4 rows
            bool all_same = have && batch_fast;
#pragma unroll
            for (int u = 0; u < kZhUnroll; ++u)
                all_same = all_same && (z[u].v[0] == cur_z) && (z[u].v[1] == cur_z) && (z[u].v[2] == cur_z) &&
                           (z[u].v[3] == cur_z);
            if (__all_sync(0xffffffffu, all_same)) {
                if (cur_ok) {
#pragma unroll
                    for (int u = 0; u < kZhUnroll; ++u) zh_add4<VT>(run, v[u].v, a, ZP ? cur_p : a.pivot);
                }
                continue;
            }
            // ---- otherwise ONE copy of the row code walks the batch (it used to be unrolled four times,
            // with the flush code inlined in each: on irregular zones the kernel's top stall was
            // `no_instruction`, 6 cycles per issued instruction -- instruction-cache misses)
            static_assert(kZhUnroll == 4, "the row pick below is written for 4 rows");
#pragma unroll 1
            for (int u = 0; u < kZhUnroll; ++u) {
                const ZhQuad<VT> vq = u == 0 ? v[0] : (u == 1 ? v[1] : (u == 2 ? v[2] : v[3]));
                const ZhQuad<ZT> zq = u == 0 ? z[0] : (u == 1 ? z[1] : (u == 2 ? z[2] : z[3]));
                const int nvu = batch_fast ? 4 : ((y + u < y1) ? nv : 0);
                const bool same = have && (zq.v[0] == cur_z) && (zq.v[1] == cur_z) && (zq.v[2] == cur_z) &&
                                  (zq.v[3] == cur_z);
                const bool fast = (nvu == 4) && same;
                if (!__all_sync(0xffffffffu, fast || nvu == 0)) {
                    // Some lane meets a zone boundary (or a ragged right edge).  A boundary between two
                    // raster ROWS reaches every lane at the row's first cell: that cell is handled with the
                    // collective flush (all 32 lanes take part; lanes leaving the same zone combine their
                    // runs by shuffles).  A boundary between two COLUMNS wanders through single lanes: the
                    // other three cells are each lane's own business -- no votes, no shuffles, a lane that
                    // changes zone flushes its own run (round 2 voted once per cell of such a row).
                    auto enter = [&](ZT zk) {
                        cur_z = zk;
                        have = (zk == zk);
                        cur_ok = zh_key<ZT>(zk, cur_key);
                        if constexpr (sizeof(ZT) == 8 && ZT(0.5) == ZT(0)) {
                            if (!cur_ok && a.sentinel != nullptr) *a.sentinel = 1;
                        }
                        if constexpr (ZP) {
                            if (cur_ok) {
                                const int ps = zh_find(a.keys, a.cap, cur_key);
                                cur_p = ps >= 0 ? a.zone_pivots[ps] : a.pivot;
                            }
                        }
                    };
                    {
                        const bool live = 0 < nvu;
                        const ZT zk = zq.v[0];
                        const bool change = live && (!have || !(zk == cur_z));
                        if (__any_sync(0xffffffffu, change)) flush_all(change && have);
                        if (change) enter(zk);
                        if (live && cur_ok) zh_add<VT>(run, vq.v[0], a, ZP ? cur_p : a.pivot);
                    }
#pragma unroll 1
                    for (int k = 1; k < 4; ++k) {
                        if (k < nvu) {
                            const ZT zk = k == 1 ? zq.v[1] : (k == 2 ? zq.v[2] : zq.v[3]);
                            const VT vk = k == 1 ? vq.v[1] : (k == 2 ? vq.v[2] : vq.v[3]);
                            if (!have || !(zk == cur_z)) {
                                if (have && cur_ok) {
                                    const double mn = sizeof(VT) == 4 ? (double)run.mnf : run.mnd;
                                    const double mx = sizeof(VT) == 4 ? (double)run.mxf : run.mxd;
                                    merge(cur_key, run.cnt, run.s1, run.s2, mn, mx);
                                    zh_reset<VT>(run);
                                }
                                enter(zk);
                            }
                            if (cur_ok) zh_add<VT>(run, vk, a, ZP ? cur_p : a.pivot);
                        }
                    }
                    __syncwarp();
                } else if (fast && cur_ok) {
                    zh_add4<VT>(run, vq.v, a, ZP ? cur_p : a.pivot);
                }
            }
        }
    }
    flush_all(have);
    __syncthreads();
    for (int i = threadIdx.x; i < kCap; i += blockDim.x) {
        const long long key = s_keys[i];
        if (key != kZhEmpty) {
            const int s = zh_slot(a.keys, a.cap, key, a.cap);
            if (s < 0) { *a.overflow = 1; continue; }
            if (s_cnt[i] == 0u) continue;
            atomicAdd(&a.count[s], (unsigned long long)s_cnt[i]);
            atomicAdd(&a.s1[s], s_s1[i]);
            atomicAdd(&a.s2[s], s_s2[i]);
            if constexpr (sizeof(VT) == 4) {
                zh_atomic_min(&a.vmin[s], (double)zh_funkey(s_mn[i]));
                zh_atomic_max(&a.vmax[s], (double)zh_funkey(s_mx[i]));
            } else {
                zh_atomic_min(&a.vmin[s], s_mn[i]);
                zh_atomic_max(&a.vmax[s], s_mx[i]);
            }
        }
    }
}

// ----------------------------------------------------------------------------- majority
// `majority` (zonal.py:56-68: np.unique(values, return_counts) -> the most frequent value, the
// smallest one on ties) needs per-zone value histograms.  One pass counts (zone, value) PAIRS in
// the same kind of hash table: key = (int32 zone id << 32) | (float32 bit pattern of the value ^
// kZpValueXor).  The XOR moves the empty key kZhEmpty = (INT32_MIN << 32) | 0 onto the pair (zone
// INT32_MIN, quiet NaN), which is never counted; with the plain bit pattern it was the pair (INT32_MIN,
// 0.0) -- the usual int32 nodata zone and a common value -- and that pair's counts landed in an "empty"
// slot.  The host then picks, per zone, the value with the largest count.  Meant for categorical
// value rasters (few distinct values per zone); `cap` bounds the number of distinct pairs.
constexpr unsigned kZpValueXor = 0x7fc00000u;
struct ZpArgs {
    const float *values;
    const int *zones;
    int64_t n, W;
    int has_nodata;
    float nodata;
    long long *keys;
    unsigned long long *count;
    int cap;
    int *overflow;
};

__global__ void __launch_bounds__(kZhThreads) zonal_pair_kernel(const __grid_constant__ ZpArgs a) {
    __shared__ long long s_keys[kZhLocalCap * 2];
    __shared__ unsigned s_cnt[kZhLocalCap * 2];
    constexpr int kCap = kZhLocalCap * 2;
    for (int i = threadIdx.x; i < kCap; i += blockDim.x) { s_keys[i] = kZhEmpty; s_cnt[i] = 0u; }
    __syncthreads();
    const bool al = ((reinterpret_cast<uintptr_t>(a.values) | reinterpret_cast<uintptr_t>(a.zones)) & 15) == 0 &&
                    (a.W % 4 == 0);
    // Every lane keeps TWO open runs (zone, value, count): class boundaries on a real categorical raster
    // are noisy -- a lane walking down its 4 columns flips between the two classes either side of a
    // boundary many times before it leaves it behind -- so a single run was flushed at every flip (a vote
    // and a shuffle per cell of such a row, 43 instructions per cell).  Now:
    //   * clean batch (one vote per 4 rows): every cell of every lane lies in the lane's zone and holds
    //     one of the lane's two values -> per cell two float compares and two adds, nothing else (an
    //     invalid cell -- NaN, inf, nodata -- matches neither value, so validity needs no test here);
    //   * anything else: ONE copy of the generic per-lane code walks the batch's rows cell by cell; a third
    //     pair evicts the run used less recently.  No votes, no shuffles: a flush is the lane's own
    //     business (native 32-bit shared-memory atomics), and the code stays small enough for the
    //     instruction cache (ncu of the unrolled version: `no_instruction` among the top stalls).
    int zone0 = 0, zone1 = 0;
    float v0 = nan_of<float>(), v1 = nan_of<float>();   // NaN never matches: the runs start empty
    unsigned c0 = 0u, c1 = 0u;
    bool last1 = false;      // the run used most recently is run 1
    auto merge = [&](int zone, float val, unsigned cnt) {
        const long long key = ((long long)zone << 32) | (long long)(__float_as_uint(val) ^ kZpValueXor);
        int s = zh_slot(s_keys, kCap, key, 64);
        if (s >= 0) { atomicAdd(&s_cnt[s], cnt); return; }
        s = zh_slot(a.keys, a.cap, key, a.cap);
        if (s < 0) *a.overflow = 1; else atomicAdd(&a.count[s], (unsigned long long)cnt);
    };
    const int lane = threadIdx.x & 31;
    const int64_t H = a.n / a.W;
    const int64_t n_strips = (a.W + 127) / 128, n_segs = (H + kZhSegRows - 1) / kZhSegRows;
    const int64_t warps_total = (int64_t)gridDim.x * (kZhThreads / 32);
    static_assert(kZhUnroll == 4, "the row pick below is written for 4 rows");
    for (int64_t task = (int64_t)blockIdx.x * (kZhThreads / 32) + (threadIdx.x >> 5); task < n_strips * n_segs;
         task += warps_total) {
        const int64_t seg = task / n_strips, strip = task % n_strips;
        const int64_t x = strip * 128 + 4 * lane;
        const int64_t y0 = seg * kZhSegRows, y1 = min(y0 + (int64_t)kZhSegRows, H);
        const int nv = (int)max((int64_t)0, min((int64_t)4, a.W - x));
        for (int64_t y = y0; y < y1; y += kZhUnroll) {
            ZhQuad<float> v[kZhUnroll];
            ZhQuad<int> z[kZhUnroll];
#pragma unroll
            for (int u = 0; u < kZhUnroll; ++u) {
                const int64_t i0 = (y + u) * a.W + x;
                const int nvu = (y + u < y1) ? nv : 0;
                v[u] = zh_load<float>(a.values, i0, i0 + nvu, al);
                z[u] = zh_load<int>(a.zones, i0, i0 + nvu, al);
            }
            // ---- clean batch?
            const bool full_batch = (nv == 4) && (y + kZhUnroll <= y1);
            const int zc = last1 ? zone1 : zone0;          // the zone of the run used last
            unsigned m0 = 0u, m1 = 0u;
            int zdiff = 0;
#pragma unroll
            for (int u = 0; u < kZhUnroll; ++u) {
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    zdiff |= z[u].v[k] ^ zc;
                    m0 += (v[u].v[k] == v0) ? 1u : 0u;
                    m1 += (v[u].v[k] == v1) ? 1u : 0u;
                }
            }
            if (zone0 != zc) m0 = 0u;      // a run left over from another zone takes no part
            if (zone1 != zc) m1 = 0u;
            const bool clean = full_batch && zdiff == 0 && (m0 + m1 == 4u * kZhUnroll);
            if (__all_sync(0xffffffffu, clean || nv == 0)) {
                if (nv != 0) {
                    c0 += m0;
                    c1 += m1;
                    last1 = (zone1 == zc) && (v[kZhUnroll - 1].v[3] == v1);
                }
                continue;
            }
            // ---- generic: row by row, cell by cell, every lane on its own
#pragma unroll 1
            for (int u = 0; u < kZhUnroll; ++u) {
                const ZhQuad<float> vq = u == 0 ? v[0] : (u == 1 ? v[1] : (u == 2 ? v[2] : v[3]));
                const ZhQuad<int> zq = u == 0 ? z[0] : (u == 1 ? z[1] : (u == 2 ? z[2] : z[3]));
                const int nvu = (y + u < y1) ? nv : 0;
#pragma unroll 1
                for (int k = 0; k < 4; ++k) {
                    if (k >= nvu) break;
                    const float fr = k == 0 ? vq.v[0] : (k == 1 ? vq.v[1] : (k == 2 ? vq.v[2] : vq.v[3]));
                    const int zk = k == 0 ? zq.v[0] : (k == 1 ? zq.v[1] : (k == 2 ? zq.v[2] : zq.v[3]));
                    const float f = fr + 0.0f;  // -0.0 -> +0.0: one value for np.unique
                    if (!(fabsf(f) <= 3.402823466e38f) || (a.has_nodata && f == a.nodata)) continue;
                    if (zk == zone0 && f == v0) { c0 += 1u; last1 = false; }
                    else if (zk == zone1 && f == v1) { c1 += 1u; last1 = true; }
                    else if (last1) {            // evict run 0
                        if (c0 != 0u) merge(zone0, v0, c0);
                        zone0 = zk; v0 = f; c0 = 1u; last1 = false;
                    } else {                     // evict run 1
                        if (c1 != 0u) merge(zone1, v1, c1);
                        zone1 = zk; v1 = f; c1 = 1u; last1 = true;
                    }
                }
            }
            __syncwarp();
        }
    }
    if (c0 != 0u) merge(zone0, v0, c0);
    if (c1 != 0u) merge(zone1, v1, c1);
    __syncthreads();
    for (int i = threadIdx.x; i < kCap; i += blockDim.x) {
        if (s_keys[i] != kZhEmpty && s_cnt[i]) {
            const int s = zh_slot(a.keys, a.cap, s_keys[i], a.cap);
            if (s < 0) *a.overflow = 1; else atomicAdd(&a.count[s], (unsigned long long)s_cnt[i]);
        }
    }
}

// Empties `cap` slots: keys to the empty key unless `keys` is NULL (the second pass keeps the first pass's keys),
// counts to 0, and the sums and min / max to their identities unless `s1` is NULL (the pair table has none).
__global__ void zonal_table_init_kernel(long long *keys, unsigned long long *count, double *s1, double *s2,
                                        double *vmin, double *vmax, int cap) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cap) return;
    if (keys) keys[i] = kZhEmpty;
    count[i] = 0ull;
    if (s1) { s1[i] = 0.0; s2[i] = 0.0; vmin[i] = INFINITY; vmax[i] = -INFINITY; }
}

// ---- one-call front end: pivot sampling, table compaction and header, all on the device ----------
// median of up to 4096 finite samples taken at a regular stride: a shift that keeps sum((v - p)^2)
// well conditioned (any value works; it only has to be the same for every cell).  The median, not the
// mean: one FLT_MAX-style nodata sentinel among the samples would move the mean to ~1e35, and every
// ordinary zone would then lose its values to the rounding of v - p.
template <typename VT>
__global__ void __launch_bounds__(256) zonal_pivot_kernel(const VT *__restrict__ v, int64_t n, double *out) {
    constexpr int kS = 4096;
    __shared__ double s_v[kS];
    __shared__ unsigned s_cnt;
    if (threadIdx.x == 0) s_cnt = 0u;
    __syncthreads();
    const int64_t samples = n < kS ? n : kS;
    const int64_t step = n / samples;
    for (int i = threadIdx.x; i < kS; i += 256) {
        const double x = i < samples ? (double)v[i * step] : INFINITY;
        const bool fin = fabs(x) <= 1.7976931348623157e308;
        s_v[i] = fin ? x : INFINITY;            // non-finite samples sort to the end
        if (fin) atomicAdd(&s_cnt, 1u);
    }
    __syncthreads();
    for (int k = 2; k <= kS; k <<= 1) {         // bitonic sort, ascending
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < kS; i += 256) {
                const int l = i ^ j;
                if (l > i) {
                    const double a = s_v[i], b = s_v[l];
                    if (((i & k) == 0) == (a > b)) { s_v[i] = b; s_v[l] = a; }
                }
            }
            __syncthreads();
        }
    }
    if (threadIdx.x == 0) *out = s_cnt ? s_v[s_cnt / 2] : 0.0;
}

// used slots -> dense rows of `packed` (6 rows of max_out doubles after a kZhHeader-double header), any order
constexpr int kZhHeader = 4;
__global__ void __launch_bounds__(256) zonal_compact_kernel(const long long *keys, const unsigned long long *count,
                                                            const double *s1, const double *s2, const double *vmin,
                                                            const double *vmax, int cap, double *packed, int max_out,
                                                            int *flags) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cap) return;
    const long long k = keys[i];
    if (k == kZhEmpty) return;
    const int pos = atomicAdd(&flags[1], 1);
    if (pos >= max_out) return;
    double *row = packed + kZhHeader;
    row[pos] = __longlong_as_double(k);
    row[max_out + pos] = __longlong_as_double((long long)count[i]);
    row[2 * max_out + pos] = s1[i];
    row[3 * max_out + pos] = s2[i];
    row[4 * max_out + pos] = vmin[i];
    row[5 * max_out + pos] = vmax[i];
}
__global__ void zonal_header_kernel(double *packed, const int *flags, const double *pivot) {
    packed[0] = (double)flags[1];   // used slots
    packed[1] = (double)flags[0];   // table overflow
    packed[2] = *pivot;
    packed[3] = (double)flags[2];   // an INT64_MIN zone was met (not in the table)
}
__global__ void zonal_flags_kernel(int *flags, double *pivot_dev, double pivot_hint) {
    flags[0] = 0;
    flags[1] = 0;
    flags[2] = 0;
    if (pivot_dev) *pivot_dev = pivot_hint;
}

// CTAs that give every warp of a zonal kernel a task: 128-column x kZhSegRows-row tasks, 8 warps per CTA
static int64_t zh_ctas_for_tasks(int64_t n, int64_t W) {
    const int64_t n_tasks = ((W + 127) / 128) * ((n / W + kZhSegRows - 1) / kZhSegRows);
    return (n_tasks + kZhThreads / 32 - 1) / (kZhThreads / 32);
}

// zonal_hash_kernel for one pass: as many CTAs as fit (no cap per SM), no more than there are tasks
template <typename VT, typename ZT> static int launch_zh(const ZhArgs &a, bool second, cudaStream_t s) {
    const auto kernel = second ? &zonal_hash_kernel<VT, ZT, true> : &zonal_hash_kernel<VT, ZT, false>;
    constexpr size_t smem = ZhTable<VT>::kBytes;
    int64_t grid;
    if (const int rc = resident_ctas(kernel, kZhThreads, smem, INT_MAX, &grid)) return rc;
    grid = std::max<int64_t>(1, std::min(grid, zh_ctas_for_tasks(a.n, a.W)));
    return launch(kernel, grid, kZhThreads, smem, s, kZonalHash, a);
}
template <typename VT> static int launch_zh(const ZhArgs &a, int zones_dtype, bool second, cudaStream_t s) {
    switch (zones_dtype) {
        case XRS_I32: return launch_zh<VT, int>(a, second, s);
        case XRS_I64: return launch_zh<VT, long long>(a, second, s);
        case XRS_F32: return launch_zh<VT, float>(a, second, s);
        default: return launch_zh<VT, double>(a, second, s);
    }
}

// The used slots and the pass's flags into `packed` (layout in xrs_b200.h).
static int zh_compact(const ZhArgs &a, double *packed, int max_out, int *flags, cudaStream_t s) {
    zonal_compact_kernel<<<(a.cap + 255) / 256, 256, 0, s>>>(a.keys, a.count, a.s1, a.s2, a.vmin, a.vmax, a.cap, packed,
                                                             max_out, flags);
    zonal_header_kernel<<<1, 1, 0, s>>>(packed, flags, packed + 2);
    XRS_CUDA(cudaGetLastError());
    return XRS_OK;
}

// One group-by pass with everything it enqueues.  First pass: samples the pivot (unless use_pivot_hint) and
// empties the table.  Second pass: resets the accumulators, keeps the first pass's keys and sums about
// zone_pivots[slot].  Then both accumulate and compact.
static int zh_pass(bool second, const void *values, int values_dtype, const void *zones, int zones_dtype, int64_t n,
                   int64_t row_len, int has_nodata, double nodata, int use_pivot_hint, double pivot_hint,
                   const double *zone_pivots, int64_t *keys, int64_t *count, double *s1, double *s2, double *vmin,
                   double *vmax, int cap, double *packed, int max_out, int *flags, cudaStream_t st) {
    XRS_REQUIRE(values && zones && keys && count && s1 && s2 && vmin && vmax && packed && flags &&
                    (zone_pivots || !second),
                "NULL pointer");
    XRS_REQUIRE(values_dtype == XRS_F32 || values_dtype == XRS_F64, "values must be float32 or float64");
    XRS_REQUIRE(zones_dtype >= XRS_F32 && zones_dtype <= XRS_I64, "unknown zones dtype");
    XRS_REQUIRE(cap >= 1024 && (cap & (cap - 1)) == 0, "cap must be a power of two >= 1024");
    XRS_REQUIRE(max_out >= 1, "max_out must be positive");
    XRS_REQUIRE(n >= 1 && row_len >= 1 && n % row_len == 0, "n must be a positive multiple of row_len");
    double *pivot_dev = packed + 2;   // the header's pivot cell doubles as the device-side pivot
    zonal_flags_kernel<<<1, 1, 0, st>>>(flags, pivot_dev, pivot_hint);
    if (!use_pivot_hint) {
        if (values_dtype == XRS_F32) zonal_pivot_kernel<float><<<1, 256, 0, st>>>((const float *)values, n, pivot_dev);
        else zonal_pivot_kernel<double><<<1, 256, 0, st>>>((const double *)values, n, pivot_dev);
    }
    zonal_table_init_kernel<<<(cap + 255) / 256, 256, 0, st>>>(second ? nullptr : (long long *)keys,
                                                               (unsigned long long *)count, s1, s2, vmin, vmax, cap);
    XRS_CUDA(cudaGetLastError());
    ZhArgs a;
    a.values = values; a.zones = zones; a.n = n; a.W = row_len;
    a.pivot = 0.0; a.pivot_ptr = second ? nullptr : pivot_dev; a.zone_pivots = zone_pivots;
    a.has_nodata = has_nodata; a.nodata = nodata;
    a.keys = (long long *)keys; a.count = (unsigned long long *)count; a.s1 = s1; a.s2 = s2; a.vmin = vmin;
    a.vmax = vmax; a.cap = cap; a.overflow = flags; a.sentinel = flags + 2;
    const int rc = values_dtype == XRS_F32 ? launch_zh<float>(a, zones_dtype, second, st)
                                           : launch_zh<double>(a, zones_dtype, second, st);
    if (rc != XRS_OK) return rc;
    return zh_compact(a, packed, max_out, flags, st);
}

}  // namespace xrs

using namespace xrs;

extern "C" {

int xrs_zonal_hash_run(const void *values, int values_dtype, const void *zones, int zones_dtype, int64_t n,
                       int64_t row_len, int has_nodata, double nodata, int use_pivot_hint, double pivot_hint,
                       int64_t *keys, int64_t *count, double *s1, double *s2, double *vmin, double *vmax, int cap,
                       double *packed, int max_out, int *flags, xrs_stream_t s) {
    return zh_pass(false, values, values_dtype, zones, zones_dtype, n, row_len, has_nodata, nodata, use_pivot_hint,
                   pivot_hint, nullptr, keys, count, s1, s2, vmin, vmax, cap, packed, max_out, flags, (cudaStream_t)s);
}

int xrs_zonal_hash_second_pass(const void *values, int values_dtype, const void *zones, int zones_dtype, int64_t n,
                               int64_t row_len, int has_nodata, double nodata, const int64_t *keys,
                               const double *zone_pivots, int64_t *count, double *s1, double *s2, double *vmin,
                               double *vmax, int cap, double *packed, int max_out, int *flags, xrs_stream_t s) {
    // every key of this raster is already in the table: the kernel's find-or-insert only finds
    return zh_pass(true, values, values_dtype, zones, zones_dtype, n, row_len, has_nodata, nodata, 1, 0.0,
                   zone_pivots, (int64_t *)keys, count, s1, s2, vmin, vmax, cap, packed, max_out, flags,
                   (cudaStream_t)s);
}

int xrs_zonal_pair_count(const float *values, const int32_t *zones, int64_t n, int64_t row_len, int has_nodata,
                         double nodata, int64_t *keys, int64_t *count, int cap, int *overflow, xrs_stream_t s) {
    XRS_REQUIRE(keys && count && overflow, "NULL pointer");
    XRS_REQUIRE(cap >= 1024 && (cap & (cap - 1)) == 0, "cap must be a power of two >= 1024");
    cudaStream_t st = (cudaStream_t)s;
    // the table is emptied also for an empty raster: the caller reads its keys back
    zonal_table_init_kernel<<<(cap + 255) / 256, 256, 0, st>>>((long long *)keys, (unsigned long long *)count, nullptr,
                                                               nullptr, nullptr, nullptr, cap);
    XRS_CUDA(cudaMemsetAsync(overflow, 0, sizeof(int), st));
    if (n <= 0) return XRS_OK;
    XRS_REQUIRE(values && zones, "NULL pointer");
    XRS_REQUIRE(row_len >= 1 && n % row_len == 0, "n must be a multiple of row_len");
    ZpArgs a;
    a.values = values; a.zones = (const int *)zones; a.n = n; a.W = row_len; a.has_nodata = has_nodata;
    a.nodata = (float)nodata; a.keys = (long long *)keys; a.count = (unsigned long long *)count; a.cap = cap;
    a.overflow = overflow;
    const int64_t grid = std::max<int64_t>(1, std::min((int64_t)sm_count() * 4, zh_ctas_for_tasks(n, row_len)));
    return launch(zonal_pair_kernel, grid, kZhThreads, 0, st, kZonalPair, a);
}

}  // extern "C"

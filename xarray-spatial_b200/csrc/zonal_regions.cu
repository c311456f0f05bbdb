// zonal_regions.cu -- zonal.regions (zonal.py:1406-1549) as a union-find over the per-cell rule of
// zonal_regions_rule.cuh, and the bounds pass of zonal.trim / zonal.crop (zonal.py:1651-1940).
//
// regions: a code pass reads the raster once and writes each cell's match bits and new-uid flag; a count and a
// scan number the new-uid cells; each 32 x 32 tile unions its own edges in shared memory and writes its cells'
// local roots; the edges that cross tiles (only cells on a tile's outer ring make them) are unioned with global
// atomics that always hang the larger root under the smaller (Playne & Hawick 2018, Allegretti et al. 2019); the
// label pass writes uid[root].  Roots are the lowest index of their component, so the result does not depend on
// the order of the unions.  Indices are int32 below 2^31 cells and int64 above (DESIGN.md section 4.12).
#include "common.cuh"
#include "zonal_regions_rule.cuh"

namespace xrs {
namespace {

using namespace zr;

constexpr int kTile = 32;                // union tile side
constexpr int kTileThreads = 256;
constexpr int kScanThreads = 256;
constexpr int kScanPer = 16;             // cells per thread of the numbering passes
constexpr int64_t kScanChunk = (int64_t)kScanThreads * kScanPer;

__device__ __forceinline__ int ld_cg(const int *p) { return __ldcg(p); }
__device__ __forceinline__ long long ld_cg(const long long *p) { return __ldcg(p); }

template <typename Idx> __device__ Idx find_root(const Idx *p, Idx x) {
    Idx q = ld_cg(p + x);
    while (q != x) {
        x = q;
        q = ld_cg(p + x);
    }
    return x;
}

// Lock-free union: the larger root goes under the smaller; a lost race continues with the root it lost to.
template <typename Idx> __device__ void unite(Idx *p, Idx a, Idx b) {
    while (true) {
        a = find_root(p, a);
        b = find_root(p, b);
        if (a == b) return;
        if (a > b) {
            const Idx t = a;
            a = b;
            b = t;
        }
        const Idx old = atomicMin(p + b, a);
        if (old == b) return;
        b = old;
    }
}

__device__ int find_shared(volatile int *p, int x) {
    int q = p[x];
    while (q != x) {
        x = q;
        q = p[x];
    }
    return x;
}

__device__ void unite_shared(int *p, int a, int b) {
    while (true) {
        a = find_shared(p, a);
        b = find_shared(p, b);
        if (a == b) return;
        if (a > b) {
            const int t = a;
            a = b;
            b = t;
        }
        const int old = atomicMin(p + b, a);
        if (old == b) return;
        b = old;
    }
}

template <typename T> __global__ void zr_code_kernel(Cells<T> z, int n, int64_t H, int64_t W, uint16_t *code) {
    const int64_t N = H * W;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < N; k += (int64_t)gridDim.x * blockDim.x)
        code[k] = (uint16_t)cell_code<T>(n, H, W, k / W, k % W, z);
}

// Exclusive scan of one value per thread over the block; returns the block's total in *total.
template <typename Idx> __device__ Idx block_exclusive_scan(Idx v, Idx *total) {
    __shared__ Idx warp_sums[kScanThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    Idx incl = v;
    for (int d = 1; d < 32; d <<= 1) {
        const Idx o = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += o;
    }
    if (lane == 31) warp_sums[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        Idx w = lane < kScanThreads / 32 ? warp_sums[lane] : 0;
        for (int d = 1; d < 32; d <<= 1) {
            const Idx o = __shfl_up_sync(0xffffffffu, w, d);
            if (lane >= d) w += o;
        }
        if (lane < kScanThreads / 32) warp_sums[lane] = w;
    }
    __syncthreads();
    const Idx before = warp ? warp_sums[warp - 1] : 0;
    *total = warp_sums[kScanThreads / 32 - 1];
    __syncthreads();
    return before + incl - v;
}

// New-uid count of each kScanChunk-cell chunk.
template <typename Idx> __global__ void zr_count_kernel(const uint16_t *code, int64_t N, Idx *sums) {
    const int64_t base = (int64_t)blockIdx.x * kScanChunk + (int64_t)threadIdx.x * kScanPer;
    Idx c = 0;
    for (int i = 0; i < kScanPer; ++i)
        if (base + i < N && (code[base + i] & kNew)) ++c;
    Idx total;
    block_exclusive_scan<Idx>(c, &total);
    if (threadIdx.x == 0) sums[blockIdx.x] = total;
}

// Exclusive scan of the chunk counts in place, by one block.
template <typename Idx> __global__ void zr_scan_sums_kernel(Idx *sums, int64_t nb) {
    Idx carry = 0;
    for (int64_t b0 = 0; b0 < nb; b0 += kScanThreads) {
        const int64_t b = b0 + threadIdx.x;
        const Idx v = b < nb ? sums[b] : 0;
        Idx total;
        const Idx ex = block_exclusive_scan<Idx>(v, &total);
        if (b < nb) sums[b] = carry + ex;
        carry += total;
    }
}

// uid[k]: the number of new-uid cells at or before k.
template <typename Idx> __global__ void zr_uid_kernel(const uint16_t *code, int64_t N, const Idx *sums, Idx *uid) {
    const int64_t base = (int64_t)blockIdx.x * kScanChunk + (int64_t)threadIdx.x * kScanPer;
    Idx c = 0;
    for (int i = 0; i < kScanPer; ++i)
        if (base + i < N && (code[base + i] & kNew)) ++c;
    Idx total;
    Idx u = sums[blockIdx.x] + block_exclusive_scan<Idx>(c, &total);
    for (int i = 0; i < kScanPer && base + i < N; ++i) {
        if (code[base + i] & kNew) ++u;
        uid[base + i] = u;
    }
}

__device__ __forceinline__ bool same_tile(int64_t a, int64_t b, int64_t W) {
    return (a / W) / kTile == (b / W) / kTile && (a % W) / kTile == (b % W) / kTile;
}

// Each tile unions the edges of its cells whose ends both lie in it, then points every cell at its tile-local root (the
// lowest global index of its tile-local component: row-major order within a tile is the global order).
template <typename Idx>
__global__ void __launch_bounds__(kTileThreads)
    zr_tile_kernel(const uint16_t *code, int n, int64_t H, int64_t W, int64_t tiles_x, int64_t n_tiles, Idx *parent) {
    __shared__ int lp[kTile * kTile];
    for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const int64_t y0 = (t / tiles_x) * kTile, x0 = (t % tiles_x) * kTile;
        for (int i = threadIdx.x; i < kTile * kTile; i += kTileThreads) lp[i] = i;
        __syncthreads();
        for (int i = threadIdx.x; i < kTile * kTile; i += kTileThreads) {
            const int64_t y = y0 + i / kTile, x = x0 + i % kTile;
            if (y >= H || x >= W) continue;
            for_each_edge(n, H, W, y, x, code[y * W + x], [&](int64_t a, int64_t b) {
                const int64_t ay = a / W - y0, ax = a % W - x0, by = b / W - y0, bx = b % W - x0;
                if (ay < 0 || ay >= kTile || ax < 0 || ax >= kTile || by < 0 || by >= kTile || bx < 0 ||
                    bx >= kTile)
                    return;
                unite_shared(lp, (int)(ay * kTile + ax), (int)(by * kTile + bx));
            });
        }
        __syncthreads();
        for (int i = threadIdx.x; i < kTile * kTile; i += kTileThreads) {
            const int64_t y = y0 + i / kTile, x = x0 + i % kTile;
            if (y >= H || x >= W) continue;
            const int r = find_shared(lp, i);
            parent[y * W + x] = (Idx)((y0 + r / kTile) * W + x0 + r % kTile);
        }
        __syncthreads();
    }
}

// The edges the tiles left: those of a cell on its tile's outer ring, the only cells whose windows reach into
// another tile, that do not lie wholly in the cell's own tile.  That includes an edge between two slots in one
// neighbouring tile (8-neighbourhood: the three slots left of a cell on the tile's left edge).
template <typename Idx> __global__ void zr_border_kernel(const uint16_t *code, int n, int64_t H, int64_t W, Idx *parent) {
    const int64_t N = H * W;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < N; k += (int64_t)gridDim.x * blockDim.x) {
        const int64_t y = k / W, x = k % W;
        const int ly = (int)(y % kTile), lx = (int)(x % kTile);
        if (ly != 0 && ly != kTile - 1 && lx != 0 && lx != kTile - 1) continue;
        for_each_edge(n, H, W, y, x, code[k], [&](int64_t a, int64_t b) {
            if (!same_tile(a, k, W) || !same_tile(b, k, W)) unite<Idx>(parent, (Idx)a, (Idx)b);
        });
    }
}

template <typename T, typename OutT, typename Idx>
__global__ void zr_label_kernel(const uint16_t *code, const Idx *parent, const Idx *uid, int64_t H, int64_t W,
                                char *out, int64_t out_pitch) {
    const int64_t N = H * W;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < N; k += (int64_t)gridDim.x * blockDim.x) {
        const int64_t y = k / W, x = k % W;
        OutT *row = reinterpret_cast<OutT *>(out + y * out_pitch);
        if constexpr (std::is_floating_point_v<T>) {
            if (code[k] & kNan) {
                row[x] = (OutT)NAN;
                continue;
            }
        }
        Idx r = (Idx)k, q = parent[r];
        while (q != r) {
            r = q;
            q = parent[r];
        }
        row[x] = (OutT)(int64_t)uid[r];   // int64 labels cast once, to the cell type (bool: all true)
    }
}

bool wide_index(int64_t N) { return N > (int64_t)INT32_MAX; }

int64_t regions_need(int64_t H, int64_t W) {
    const int64_t N = H * W, idx = wide_index(N) ? 8 : 4, nb = (N + kScanChunk - 1) / kScanChunk;
    return align256(2 * N) + 2 * align256(idx * N) + align256(idx * (nb + 1));
}

int64_t grid_for(int64_t work, int threads) {
    int64_t g = (work + threads - 1) / threads;
    const int64_t cap = (int64_t)sm_count() * 32;
    return g < 1 ? 1 : (g > cap ? cap : g);
}

template <typename T, typename OutT, typename Idx>
int regions_run(const void *in, int64_t in_pitch, int64_t H, int64_t W, int n, void *out, int64_t out_pitch,
                char *scratch, cudaStream_t s) {
    const int64_t N = H * W, nb = (N + kScanChunk - 1) / kScanChunk;
    uint16_t *code = (uint16_t *)scratch;
    Idx *parent = (Idx *)(scratch + align256(2 * N));
    Idx *uid = (Idx *)((char *)parent + align256((int64_t)sizeof(Idx) * N));
    Idx *sums = (Idx *)((char *)uid + align256((int64_t)sizeof(Idx) * N));
    const Cells<T> z{(const char *)in, in_pitch};
    zr_code_kernel<T><<<(unsigned)grid_for(N, 256), 256, 0, s>>>(z, n, H, W, code);
    XRS_CUDA(cudaGetLastError());
    zr_count_kernel<Idx><<<(unsigned)nb, kScanThreads, 0, s>>>(code, N, sums);
    XRS_CUDA(cudaGetLastError());
    zr_scan_sums_kernel<Idx><<<1, kScanThreads, 0, s>>>(sums, nb);
    XRS_CUDA(cudaGetLastError());
    zr_uid_kernel<Idx><<<(unsigned)nb, kScanThreads, 0, s>>>(code, N, sums, uid);
    XRS_CUDA(cudaGetLastError());
    const int64_t tiles_x = (W + kTile - 1) / kTile, n_tiles = tiles_x * ((H + kTile - 1) / kTile);
    const int64_t tile_grid = n_tiles < (int64_t)sm_count() * 64 ? n_tiles : (int64_t)sm_count() * 64;
    zr_tile_kernel<Idx><<<(unsigned)tile_grid, kTileThreads, 0, s>>>(code, n, H, W, tiles_x, n_tiles, parent);
    XRS_CUDA(cudaGetLastError());
    zr_border_kernel<Idx><<<(unsigned)grid_for(N, 256), 256, 0, s>>>(code, n, H, W, parent);
    XRS_CUDA(cudaGetLastError());
    zr_label_kernel<T, OutT, Idx><<<(unsigned)grid_for(N, 256), 256, 0, s>>>(code, parent, uid, H, W, (char *)out,
                                                                             out_pitch);
    XRS_CUDA(cudaGetLastError());
    return XRS_OK;
}

template <typename T, typename OutT = T>
int regions_typed(const void *in, int64_t in_pitch, int64_t H, int64_t W, int n, void *out, int64_t out_pitch,
                  char *scratch, cudaStream_t s) {
    if (wide_index(H * W))
        return regions_run<T, OutT, long long>(in, in_pitch, H, W, n, out, out_pitch, scratch, s);
    return regions_run<T, OutT, int>(in, in_pitch, H, W, n, out, out_pitch, scratch, s);
}

int check_shape(int64_t H, int64_t W) {
    XRS_REQUIRE(H >= 0 && W >= 0, "negative raster shape");
    XRS_REQUIRE(H < INT32_MAX && W < INT32_MAX, "rows and columns must each be below 2^31");
    XRS_REQUIRE(W == 0 || H <= ((int64_t)1 << 40) / W, "a raster of more than 2^40 cells");
    return XRS_OK;
}

// ----------------------------------------------------------------------------- trim / crop bounds
struct Targets {
    const double *dv;      // the values as float64
    const long long *iv;   // the values as int64 (int_values only)
    int nv;
    int int_values;        // every value is an integer: integer cells compare exactly
};

// numba's `==` between a cell and a value: integers exactly, anything with a float (and uint64 against an int64,
// which numba promotes to float64) in float64.  NaN never equals.
template <typename T> __device__ __forceinline__ bool equals_any(T v, const Targets &t) {
    for (int i = 0; i < t.nv; ++i) {
        if constexpr (std::is_integral_v<T> && !std::is_same_v<T, unsigned long long>) {
            if (t.int_values) {
                if ((long long)v == t.iv[i]) return true;
                continue;
            }
        }
        if ((double)v == t.dv[i]) return true;
    }
    return false;
}

constexpr int kBoundsThreads = 256;

// out4: least and largest row, least and largest column of the qualifying cells (mode 0, trim: cells equal to
// none of the values; mode 1, crop: cells equal to one of them).
template <typename T>
__global__ void __launch_bounds__(kBoundsThreads)
    zb_bounds_kernel(Cells<T> z, int64_t H, int64_t W, int mode, Targets t, long long *out4) {
    long long r0 = LLONG_MAX, r1 = -1, c0 = LLONG_MAX, c1 = -1;
    for (int64_t r = blockIdx.x; r < H; r += gridDim.x) {
        const T *row = reinterpret_cast<const T *>(z.base + r * z.pitch);
        for (int64_t c = threadIdx.x; c < W; c += kBoundsThreads) {
            const bool hit = equals_any<T>(row[c], t);
            if (hit == (mode == 1)) {
                r0 = r0 < r ? r0 : r;
                r1 = r;
                c0 = c0 < c ? c0 : c;
                c1 = c1 > c ? c1 : c;
            }
        }
    }
    for (int d = 16; d; d >>= 1) {
        r0 = min(r0, __shfl_xor_sync(0xffffffffu, r0, d));
        r1 = max(r1, __shfl_xor_sync(0xffffffffu, r1, d));
        c0 = min(c0, __shfl_xor_sync(0xffffffffu, c0, d));
        c1 = max(c1, __shfl_xor_sync(0xffffffffu, c1, d));
    }
    if ((threadIdx.x & 31) == 0 && r1 >= 0) {
        atomicMin(out4 + 0, r0);
        atomicMax(out4 + 1, r1);
        atomicMin(out4 + 2, c0);
        atomicMax(out4 + 3, c1);
    }
}

__global__ void zb_init_kernel(long long *out4) {
    out4[0] = LLONG_MAX;
    out4[1] = -1;
    out4[2] = LLONG_MAX;
    out4[3] = -1;
}

template <typename T>
int bounds_typed(const void *in, int64_t in_pitch, int64_t H, int64_t W, int mode, const Targets &t, long long *out4,
                 cudaStream_t s) {
    zb_init_kernel<<<1, 1, 0, s>>>(out4);
    XRS_CUDA(cudaGetLastError());
    if (H == 0 || W == 0) return XRS_OK;
    const int64_t cap = (int64_t)sm_count() * 16;
    zb_bounds_kernel<T><<<(unsigned)(H < cap ? H : cap), kBoundsThreads, 0, s>>>(Cells<T>{(const char *)in, in_pitch},
                                                                                H, W, mode, t, out4);
    XRS_CUDA(cudaGetLastError());
    return XRS_OK;
}

}  // namespace
}  // namespace xrs

using namespace xrs;

extern "C" int xrs_zonal_regions_scratch_bytes(int64_t H, int64_t W, int64_t *bytes) {
    XRS_REQUIRE(bytes != nullptr, "NULL pointer");
    const int rc = check_shape(H, W);
    if (rc) return rc;
    *bytes = regions_need(H, W);
    return XRS_OK;
}

extern "C" int xrs_zonal_regions(const void *in, int dtype, int64_t in_pitch, int64_t H, int64_t W, int neighborhood,
                                 void *out, int64_t out_pitch, void *scratch, int64_t scratch_bytes, xrs_stream_t s) {
    int rc = check_shape(H, W);
    if (rc) return rc;
    XRS_REQUIRE(neighborhood == 4 || neighborhood == 8, "neighborhood must be 4 or 8");
    XRS_REQUIRE(in_cell_set(kZonalCells, dtype), "unknown cell type");
    if (H == 0 || W == 0) return XRS_OK;
    XRS_REQUIRE(in && out, "NULL pointer");
    XRS_TRY(check_cells_arg(in, dtype, kZonalCells, in_pitch, W));
    XRS_TRY(check_out_pitch(out_pitch, cell_size(dtype), W));
    XRS_TRY(check_scratch(scratch, scratch_bytes, regions_need(H, W), "xrs_zonal_regions_scratch_bytes"));
    return with_cell_type(kZonalCells, dtype, [&](auto z) {
        using T = decltype(z);
        const int n = neighborhood;
        char *sc = (char *)scratch;
        if constexpr (std::is_same_v<T, bool>)   // bool cells are read as uint8 and labelled as bool
            return regions_typed<uint8_t, bool>(in, in_pitch, H, W, n, out, out_pitch, sc, (cudaStream_t)s);
        else
            return regions_typed<T>(in, in_pitch, H, W, n, out, out_pitch, sc, (cudaStream_t)s);
    });
}

extern "C" int xrs_zonal_bounds(const void *in, int dtype, int64_t in_pitch, int64_t H, int64_t W, int mode,
                                const double *values, const int64_t *int_values, int n_values, int64_t *out4,
                                xrs_stream_t s) {
    int rc = check_shape(H, W);
    if (rc) return rc;
    XRS_REQUIRE(mode == 0 || mode == 1, "mode must be 0 (trim) or 1 (crop)");
    XRS_REQUIRE(in_cell_set(kZonalCells, dtype), "unknown cell type");
    XRS_REQUIRE(n_values >= 0, "negative value count");
    XRS_REQUIRE(out4 != nullptr, "NULL pointer");
    XRS_REQUIRE(H == 0 || W == 0 || in != nullptr, "NULL pointer");
    XRS_REQUIRE(n_values == 0 || values != nullptr, "NULL values");
    if (H && W) XRS_TRY(check_cells_arg(in, dtype, kZonalCells, in_pitch, W));
    const Targets t{values, (const long long *)int_values, n_values, int_values != nullptr};
    return with_cell_type(kZonalCells, dtype, [&](auto z) {
        using T = std::conditional_t<std::is_same_v<decltype(z), bool>, uint8_t, decltype(z)>;   // bool as uint8
        return bounds_typed<T>(in, in_pitch, H, W, mode, t, (long long *)out4, (cudaStream_t)s);
    });
}

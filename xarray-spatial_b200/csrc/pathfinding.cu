// pathfinding.cu -- a_star_search (pathfinding.py:233-382) as an exact shortest-path search over the crossable
// cells (DESIGN.md section 4.9).  A mask pass marks the crossable cells; a tiled Bellman-Ford relaxation builds the
// exact field of path lengths to the goal (pathfinding_grid.cuh), round by round from the host; a walk from the
// start follows the field to the goal and writes the running sums.  The snap is an exact argmin reduction.
#include <math.h>

#include <algorithm>

#include "common.cuh"
#include "pathfinding_grid.cuh"

namespace xrs {
namespace {

using namespace pf;

constexpr int kT = 32;          // a tile is 32 x 32 cells, one thread each
constexpr int kS = kT + 2;      // with its one-cell halo
constexpr int kWin = 64;        // the walk's shared-memory window of the field
constexpr int kBatch = 16;      // relaxation rounds enqueued between two reads of the activity counters
constexpr int64_t kCtl = 256;   // control block at the start of the scratch

// Control block: the active-tile counts of a batch of rounds (slot j is round j's input), the failure flag and
// the snap's result.
struct Ctl {
    int count[kBatch + 1];
    int fail;
    unsigned long long snap_d2, snap_idx;
};
static_assert(sizeof(Ctl) <= kCtl, "control block");

struct Barriers {
    const double *v;   // DEVICE float64 values, none NaN
    int n;
};

template <typename T> __device__ __forceinline__ bool crossable(const void *in, int64_t pitch, int64_t r, int64_t c,
                                                                const Barriers &bar) {
    const double v = (double)Cells<T>{(const char *)in, pitch}(r, c);   // as NumPy compares
    if (v != v) return false;
    for (int i = 0; i < bar.n; ++i)
        if (v == bar.v[i]) return false;
    return true;
}

__device__ __forceinline__ Dist load_dist(const Dist *f, int64_t k) {
    const int2 v = __ldcg(reinterpret_cast<const int2 *>(f + k));   // one 8-byte load, from L2: other CTAs write
    return Dist{v.x, v.y};
}

__device__ __forceinline__ void store_dist(Dist *f, int64_t k, Dist d) {
    *reinterpret_cast<int2 *>(f + k) = make_int2(d.a, d.b);
}

struct Field {   // H, W and the goal's cell each fit an int (H W < 2^31)
    Dist *dist;
    const uint8_t *mask;
    int H, W;
    int conn;
    int tiles_x, tiles_y;
    int goal_r, goal_c;
};

template <typename T>
__global__ void pf_mask_kernel(const void *in, int64_t pitch, Barriers bar, Field f, uint8_t *mask) {
    const int64_t n = (int64_t)f.H * f.W;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = k / f.W, c = k - r * f.W;
        mask[k] = crossable<T>(in, pitch, r, c, bar);
        store_dist(f.dist, k, unreached());
    }
}

// One round: every CTA takes active tiles from list_in, loads each with its halo, relaxes it until it stops
// changing, writes back its own cells that dropped, and queues each neighbouring tile next to a border cell that
// dropped for the next round (stamp[] holds the last round a tile was queued for, so it is queued once).
__global__ void __launch_bounds__(kT *kT, 2) pf_relax_kernel(Field f, const int *list_in, const int *count_in,
                                                         int *list_out, int *count_out, unsigned *stamp,
                                                         unsigned next_round, int *fail) {
    __shared__ Dist sd[kS][kS];
    __shared__ int sflag[9];
    const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * kT + tx;
    const int n = *count_in;
    for (int i = blockIdx.x; i < n; i += gridDim.x) {
        const int t = list_in[i];
        const int tr = t / f.tiles_x, tc = t - tr * f.tiles_x;
        const int r0 = tr * kT, c0 = tc * kT;
        for (int k = tid; k < kS * kS; k += kT * kT) {
            const int r = r0 - 1 + k / kS, c = c0 - 1 + k % kS;
            sd[k / kS][k % kS] = (r >= 0 && r < f.H && c >= 0 && c < f.W) ? load_dist(f.dist, (int64_t)r * f.W + c)
                                                                          : unreached();
        }
        if (tid < 9) sflag[tid] = 0;
        const int r = r0 + ty, c = c0 + tx;
        const bool mine = r < f.H && c < f.W && f.mask[(int64_t)r * f.W + c];
        const bool goal = r == f.goal_r && c == f.goal_c;
        __syncthreads();
        const Dist before = sd[ty + 1][tx + 1];
        Dist d = before;
        for (int it = 0;; ++it) {
            Dist nd = d;
            if (mine)
                nd = relax(goal ? Dist{0, 0} : d, f.conn,
                           [&](int dy, int dx) { return sd[ty + 1 + dy][tx + 1 + dx]; });
            const bool dropped = less(nd, d);
            __syncthreads();   // every read of this sweep before any write
            if (dropped) {
                d = nd;
                sd[ty + 1][tx + 1] = d;
            }
            if (!__syncthreads_or(dropped)) break;
            if (it > kT * kT) {   // a tile settles within as many sweeps as it has cells
                if (tid == 0) atomicExch(fail, 1);
                break;
            }
        }
        if (!same(d, before)) {
            store_dist(f.dist, (int64_t)r * f.W + c, d);
            const int up = ty == 0, down = ty == kT - 1, left = tx == 0, right = tx == kT - 1;
            if (up) sflag[1] = 1;
            if (down) sflag[7] = 1;
            if (left) sflag[3] = 1;
            if (right) sflag[5] = 1;
            if (f.conn == 8) {
                if (up && left) sflag[0] = 1;
                if (up && right) sflag[2] = 1;
                if (down && left) sflag[6] = 1;
                if (down && right) sflag[8] = 1;
            }
        }
        __syncthreads();
        if (tid < 9 && sflag[tid]) {
            const int nr = tr + tid / 3 - 1, nc = tc + tid % 3 - 1;
            if (nr >= 0 && nr < f.tiles_y && nc >= 0 && nc < f.tiles_x) {
                const int nt = nr * f.tiles_x + nc;
                if (atomicMax(stamp + nt, next_round) < next_round) list_out[atomicAdd(count_out, 1)] = nt;
            }
        }
        __syncthreads();   // sd and sflag are reused by the next tile
    }
}

__global__ void pf_fill_nan_kernel(double *out, int64_t out_pitch, int64_t H, int64_t W) {
    const int64_t n = H * W;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = k / W;
        out[r * out_pitch + (k - r * W)] = __longlong_as_double(0x7ff8000000000000LL);   // np.nan
    }
}

// The walk, one dependent chain: thread 0 follows successor() from the start while every neighbour of its cell is
// inside the window (or outside the raster), writing each cell's running sum; then the CTA reloads the window
// around the cell it reached.  Writes nothing when the start is unreached.
__global__ void __launch_bounds__(256) pf_walk_kernel(const Dist *dist, int64_t H, int64_t W, int conn, int64_t sr,
                                                      int64_t sc, double *out, int64_t out_pitch, int *fail) {
    __shared__ Dist win[kWin][kWin];
    __shared__ int64_t s_r, s_c;
    __shared__ double s_v;
    __shared__ int s_done;
    if (threadIdx.x == 0) {
        s_r = sr;
        s_c = sc;
        s_v = 0.0;
        s_done = !reached(load_dist(dist, sr * W + sc));
        if (!s_done) out[sr * out_pitch + sc] = 0.0;
    }
    for (;;) {
        __syncthreads();
        if (s_done) return;
        const int64_t r0 = max((int64_t)0, min(s_r - kWin / 2, H - kWin));
        const int64_t c0 = max((int64_t)0, min(s_c - kWin / 2, W - kWin));
        for (int k = threadIdx.x; k < kWin * kWin; k += blockDim.x) {
            const int64_t r = r0 + k / kWin, c = c0 + k % kWin;
            win[k / kWin][k % kWin] = (r < H && c < W) ? load_dist(dist, r * W + c) : unreached();
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            int64_t r = s_r, c = s_c;
            double v = s_v;
            Dist d = win[r - r0][c - c0];
            for (;;) {
                if (d.a == 0 && d.b == 0) {   // the goal
                    s_done = 1;
                    break;
                }
                if (!((r == 0 || r - 1 >= r0) && (r == H - 1 || r + 1 < r0 + kWin) && (c == 0 || c - 1 >= c0) &&
                      (c == W - 1 || c + 1 < c0 + kWin)))
                    break;
                const int k = successor(d, conn, [&](int dy, int dx) {
                    const int64_t rr = r + dy, cc = c + dx;
                    return (rr < 0 || rr >= H || cc < 0 || cc >= W) ? unreached() : win[rr - r0][cc - c0];
                });
                if (k < 0) {   // not a field of exact lengths: a logic error, never a valid path
                    atomicExch(fail, 1);
                    s_done = 1;
                    break;
                }
                int dy, dx;
                move(conn, k, dy, dx);
                r += dy;
                c += dx;
                d = win[r - r0][c - c0];
                v = path_value(v, dy != 0 && dx != 0);
                out[r * out_pitch + c] = v;
            }
            s_r = r;
            s_c = c;
            s_v = v;
        }
    }
}

// The snap in two passes: the least qualifying squared distance, then the least row-major index at it.
template <typename T>
__global__ void pf_snap_d2_kernel(const void *in, int64_t pitch, int64_t H, int64_t W, Barriers bar, int64_t r0,
                                  int64_t c0, unsigned long long *best) {
    const int64_t n = H * W;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = k / W, c = k - r * W, d2 = snap_d2(r, c, r0, c0);
        if (snap_qualifies(d2, H, W) && crossable<T>(in, pitch, r, c, bar)) atomicMin(best, (unsigned long long)d2);
    }
}

template <typename T>
__global__ void pf_snap_idx_kernel(const void *in, int64_t pitch, int64_t H, int64_t W, Barriers bar, int64_t r0,
                                   int64_t c0, const unsigned long long *best, unsigned long long *idx) {
    const int64_t n = H * W;
    const unsigned long long b = *best;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = k / W, c = k - r * W;
        if ((unsigned long long)snap_d2(r, c, r0, c0) == b && crossable<T>(in, pitch, r, c, bar))
            atomicMin(idx, (unsigned long long)k);
    }
}

struct Layout {
    int64_t tiles_x, tiles_y, ntiles, dist, mask, stamp, list0, list1, total;
    Layout(int64_t H, int64_t W) {
        tiles_x = (W + kT - 1) / kT;
        tiles_y = (H + kT - 1) / kT;
        ntiles = tiles_x * tiles_y;
        dist = kCtl;
        mask = dist + align256(H * W * (int64_t)sizeof(Dist));
        stamp = mask + align256(H * W);
        list0 = stamp + align256(ntiles * 4);
        list1 = list0 + align256(ntiles * 4);
        total = list1 + align256(ntiles * 4);
    }
};

int check_shape(int64_t H, int64_t W) {
    XRS_REQUIRE(H > 0 && W > 0, "a_star_search needs a raster of at least one cell");
    if (H >= kMaxCells || W >= kMaxCells || H * W >= kMaxCells) {
        set_error("a %lld x %lld raster has 2^31 cells or more; a_star_search takes fewer", (long long)H,
                  (long long)W);
        return XRS_EINVAL;
    }
    return XRS_OK;
}

int check_cells(const void *in, int in_dtype, int64_t in_pitch, int64_t W, const double *barriers, int n_barriers) {
    XRS_TRY(check_cells_arg(in, in_dtype, kRasterCells, in_pitch, W));
    XRS_REQUIRE(n_barriers >= 0 && (n_barriers == 0 || barriers != nullptr), "bad barrier list");
    return XRS_OK;
}

// The distance field from the goal: the mask pass, then batches of kBatch rounds with one read of the activity
// counts per batch.  At most H W + 1 rounds change a cell (a shortest path crosses fewer tile borders than it has
// steps), so more rounds than that is an error, never a spin.
template <typename T>
int build_field(const void *in, int64_t in_pitch, const Barriers &bar, Field f, const Layout &L, char *scratch,
                int64_t *rounds, cudaStream_t s) {
    Ctl *ctl = (Ctl *)scratch;
    uint8_t *mask = (uint8_t *)(scratch + L.mask);
    unsigned *stamp = (unsigned *)(scratch + L.stamp);
    int *lists[2] = {(int *)(scratch + L.list0), (int *)(scratch + L.list1)};
    const int64_t n = (int64_t)f.H * f.W;
    pf_mask_kernel<T><<<(unsigned)stride_grid(n), 256, 0, s>>>(in, in_pitch, bar, f, mask);
    XRS_CUDA(cudaGetLastError());
    XRS_CUDA(cudaMemsetAsync(ctl, 0, sizeof(Ctl), s));
    XRS_CUDA(cudaMemsetAsync(stamp, 0, L.ntiles * 4, s));
    // round 1 takes the goal's tile: its goal cell drops to (0, 0) there and queues what it reaches
    const int goal_tile = (int)((f.goal_r / kT) * L.tiles_x + f.goal_c / kT), one = 1;
    const unsigned first = 1;
    XRS_CUDA(cudaMemcpyAsync(lists[0], &goal_tile, 4, cudaMemcpyHostToDevice, s));
    XRS_CUDA(cudaMemcpyAsync(&ctl->count[0], &one, 4, cudaMemcpyHostToDevice, s));
    XRS_CUDA(cudaMemcpyAsync(stamp + goal_tile, &first, 4, cudaMemcpyHostToDevice, s));
    int64_t grid = 0;
    int rc = resident_ctas(pf_relax_kernel, kT * kT, 0, 2, &grid);
    if (rc) return rc;
    grid = std::min<int64_t>(grid, L.ntiles);
    const int64_t bound = n + 2;
    int64_t round = 0;   // rounds enqueued so far
    *rounds = 0;
    for (;;) {
        for (int j = 0; j < kBatch; ++j) {
            const unsigned next = (unsigned)(round + j + 2);
            pf_relax_kernel<<<(unsigned)grid, dim3(kT, kT), 0, s>>>(
                f, lists[(round + j) & 1], &ctl->count[j], lists[(round + j + 1) & 1], &ctl->count[j + 1], stamp,
                next, &ctl->fail);
            XRS_CUDA(cudaGetLastError());
        }
        Ctl h;
        XRS_CUDA(cudaMemcpyAsync(&h, ctl, sizeof(Ctl), cudaMemcpyDeviceToHost, s));
        XRS_CUDA(cudaStreamSynchronize(s));
        for (int j = 0; j < kBatch; ++j) *rounds += h.count[j] > 0;
        round += kBatch;
        if (h.fail) {
            set_error("a_star_search: a tile did not settle (internal error)");
            return XRS_ECUDA;
        }
        if (h.count[kBatch] == 0) return XRS_OK;
        if (round > bound) {
            set_error("a_star_search: the relaxation did not settle within %lld rounds (internal error)",
                      (long long)bound);
            return XRS_ECUDA;
        }
        // the last count opens the next batch; the others restart from zero
        XRS_CUDA(cudaMemsetAsync(&ctl->count[0], 0, sizeof(int) * kBatch, s));
        XRS_CUDA(cudaMemcpyAsync(&ctl->count[0], &h.count[kBatch], 4, cudaMemcpyHostToDevice, s));
        XRS_CUDA(cudaMemsetAsync(&ctl->count[kBatch], 0, sizeof(int), s));
    }
}

}  // namespace
}  // namespace xrs

using namespace xrs;

extern "C" int xrs_a_star_scratch_bytes(int64_t H, int64_t W, int64_t *bytes) {
    XRS_REQUIRE(bytes != nullptr, "NULL pointer");
    const int rc = check_shape(H, W);
    if (rc) return rc;
    *bytes = Layout(H, W).total;
    return XRS_OK;
}

extern "C" int xrs_a_star_search(const void *in, int in_dtype, int64_t in_pitch, int64_t H, int64_t W,
                                 const double *barriers, int n_barriers, int connectivity, int64_t start_row,
                                 int64_t start_col, int64_t goal_row, int64_t goal_col, double *out,
                                 int64_t out_pitch, void *scratch, int64_t scratch_bytes, int64_t *rounds,
                                 xrs_stream_t s) {
    int rc = check_shape(H, W);
    if (rc) return rc;
    rc = check_cells(in, in_dtype, in_pitch, W, barriers, n_barriers);
    if (rc) return rc;
    XRS_REQUIRE(connectivity == 4 || connectivity == 8, "connectivity must be 4 or 8");
    XRS_REQUIRE(start_row >= 0 && start_row < H && start_col >= 0 && start_col < W, "start outside the raster");
    XRS_REQUIRE(goal_row >= 0 && goal_row < H && goal_col >= 0 && goal_col < W, "goal outside the raster");
    XRS_REQUIRE(out != nullptr, "NULL output");
    XRS_TRY(check_out_pitch(out_pitch, 8, W));
    const Layout L(H, W);
    XRS_TRY(check_scratch(scratch, scratch_bytes, L.total, "xrs_a_star_scratch_bytes"));
    cudaStream_t st = (cudaStream_t)s;
    char *sc = (char *)scratch;
    const Field f{(Dist *)(sc + L.dist), (const uint8_t *)(sc + L.mask), (int)H, (int)W, connectivity,
                  (int)L.tiles_x, (int)L.tiles_y, (int)goal_row, (int)goal_col};
    const Barriers bar{barriers, n_barriers};
    int64_t nrounds = 0;
    rc = with_cell_type(kRasterCells, in_dtype, [&](auto z) {
        return build_field<decltype(z)>(in, in_pitch, bar, f, L, sc, &nrounds, st);
    });
    if (rc) return rc;
    pf_fill_nan_kernel<<<(unsigned)stride_grid(H * W), 256, 0, st>>>(out, out_pitch / 8, H, W);
    XRS_CUDA(cudaGetLastError());
    Ctl *ctl = (Ctl *)sc;
    pf_walk_kernel<<<1, 256, 0, st>>>(f.dist, H, W, connectivity, start_row, start_col, out, out_pitch / 8,
                                      &ctl->fail);
    XRS_CUDA(cudaGetLastError());
    int fail = 0;
    XRS_CUDA(cudaMemcpyAsync(&fail, &ctl->fail, 4, cudaMemcpyDeviceToHost, st));
    XRS_CUDA(cudaStreamSynchronize(st));
    if (fail) {
        set_error("a_star_search: the walk left the field of shortest lengths (internal error)");
        return XRS_ECUDA;
    }
    if (rounds) *rounds = nrounds;
    return XRS_OK;
}

extern "C" int xrs_a_star_snap(const void *in, int in_dtype, int64_t in_pitch, int64_t H, int64_t W,
                               const double *barriers, int n_barriers, int64_t row, int64_t col, int64_t *snap_row,
                               int64_t *snap_col, void *scratch, int64_t scratch_bytes, xrs_stream_t s) {
    int rc = check_shape(H, W);
    if (rc) return rc;
    rc = check_cells(in, in_dtype, in_pitch, W, barriers, n_barriers);
    if (rc) return rc;
    XRS_REQUIRE(row >= 0 && row < H && col >= 0 && col < W, "cell outside the raster");
    XRS_REQUIRE(snap_row && snap_col, "NULL pointer");
    XRS_REQUIRE(scratch != nullptr, "NULL scratch buffer");
    XRS_REQUIRE(scratch_bytes >= kCtl, "the snap needs 256 bytes of scratch");
    cudaStream_t st = (cudaStream_t)s;
    Ctl *ctl = (Ctl *)scratch;
    XRS_CUDA(cudaMemsetAsync(&ctl->snap_d2, 0xff, 16, st));
    const Barriers bar{barriers, n_barriers};
    const unsigned grid = (unsigned)stride_grid(H * W);
    rc = with_cell_type(kRasterCells, in_dtype, [&](auto z) -> int {
        using T = decltype(z);
        pf_snap_d2_kernel<T><<<grid, 256, 0, st>>>(in, in_pitch, H, W, bar, row, col, &ctl->snap_d2);
        XRS_CUDA(cudaGetLastError());
        pf_snap_idx_kernel<T><<<grid, 256, 0, st>>>(in, in_pitch, H, W, bar, row, col, &ctl->snap_d2,
                                                    &ctl->snap_idx);
        XRS_CUDA(cudaGetLastError());
        return XRS_OK;
    });
    if (rc) return rc;
    unsigned long long h[2];
    XRS_CUDA(cudaMemcpyAsync(h, &ctl->snap_d2, 16, cudaMemcpyDeviceToHost, st));
    XRS_CUDA(cudaStreamSynchronize(st));
    const bool none = h[1] == ~0ull;
    *snap_row = none ? -1 : (int64_t)(h[1] / (unsigned long long)W);
    *snap_col = none ? -1 : (int64_t)(h[1] % (unsigned long long)W);
    return XRS_OK;
}

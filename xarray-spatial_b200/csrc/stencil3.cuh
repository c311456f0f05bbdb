// stencil3.cuh -- the 3x3 "warp strip" skeleton shared by slope / aspect / curvature /
// hillshade / focal.mean / the fused surface suite.
//
// Decomposition (Hopper TMA + mbarrier pipeline, not a port of the reference's one-thread-per-cell kernels,
// slope.py:133-142): the raster is cut into CTA tiles of WARPS x 128 columns and row segments;
// a persistent CTA owns one (segment, tile) task at a time and marches down its rows.  Inside the
// tile each consumer WARP owns a 128-cell strip and each lane 4 adjacent cells (one float4), so a
// warp reads / writes 512 contiguous bytes per row.
//   * ONE producer warp per CTA streams the tile (plus a 32-byte halo each side) through a ring of
//     shared-memory stages with TMA 2-D boxes (208 cells x ROWS rows each; cp.async.bulk.tensor),
//     `full` mbarriers carry the transaction bytes, `empty` mbarriers (one arrival per consumer
//     warp) hand a stage back.  The producer is never delayed by arithmetic or stores, so the read
//     stream is steady and in raster order, and the bytes in flight per SM are set by the ring
//     (ROWS x STAGES), not by how many warps the arithmetic needs.  An earlier pipeline, where every
//     warp refilled its own 4-box ring after finishing a box, could not reach the copy rate even for
//     an operator that does nothing (the probe that compared the two, scripts/tune/tune3.cu, is in the
//     git history);
//   * out-of-raster cells are filled with NaN by the TMA unit, which is exactly the reference's
//     raster-edge rule (NaN ring for the Horn family, NaN-skipping clamped windows for focal.mean);
//   * the three input rows a cell needs are never re-read: operators keep per-row partial
//     results (column differences / weighted row sums) of the two previous rows in
//     registers and combine them with the new row ("push, then emit the row above");
//   * left / right neighbours are scalar shared-memory loads next to the lane's float4 (strip-edge
//     lanes read the neighbouring strip or the tile halo: same addresses formula);
//   * outputs go the same way in reverse: consumer lanes put their float4 into a double-buffered
//     shared-memory staging area (`out_full` / `out_empty` mbarriers), and ONE store warp writes
//     each finished tile row with a single bulk async copy (cp.async.bulk), in raster order.  The
//     earlier epilogue -- every warp storing its own 512 B per row at its own pace -- reached L2 as
//     16 pieces per tile row at 16 different times, mixed into the read stream.  Operators whose
//     staging does not fit next to the ring (the 4-output suite) keep the register stores, chosen
//     at compile time (TmaCfg::kBulk).
// Rasters TMA cannot describe (width not a multiple of 4 cells, unaligned base / pitch) run a
// per-warp ring filled by cp.async (stencil3_cpasync_kernel), which fills its ring cell by cell with
// bounds checks; the tests compare the TMA kernel with it bit for bit.  Both drive the very same
// operator code.
#pragma once
#include "common.cuh"

namespace xrs {

constexpr int kLaneCells = 4;                        // cells per lane
constexpr int kStripW = 32 * kLaneCells;             // 128 cells per warp-row
constexpr int kPad = 4;                              // pad cells each side (16 B for f32)
constexpr int kBoxW = kStripW + 2 * kPad;            // 136
constexpr int kWarpsPerCta = 8;

template <typename T> struct Vec4;  // 4 consecutive cells
template <> struct Vec4<float> { float v[4]; };
template <> struct Vec4<double> { double v[4]; };

template <typename T> __device__ __forceinline__ T shfl_up1(T v) { return __shfl_up_sync(0xffffffffu, v, 1); }
template <typename T> __device__ __forceinline__ T shfl_dn1(T v) { return __shfl_down_sync(0xffffffffu, v, 1); }

// One input row as seen by a lane: left neighbour, own 4 cells, right neighbour.
template <typename T> struct Row6 {
    T l, c[4], r;
};

// `p` points at the lane's first cell inside a shared-memory row (16-byte aligned).  The left /
// right neighbours are plain scalar loads (4-way bank conflicted, 8 extra wavefronts per
// warp-row against a budget of ~44 cycles): cheaper in issue slots than shuffles plus
// strip-edge fix-ups, and issue slots are what these kernels run out of.
template <typename T> __device__ __forceinline__ Row6<T> load_row_smem(const T *p) {
    Row6<T> o;
    if constexpr (sizeof(T) == 4) {
        const float4 q = *reinterpret_cast<const float4 *>(p);
        o.c[0] = q.x; o.c[1] = q.y; o.c[2] = q.z; o.c[3] = q.w;
    } else {
        const double2 q0 = *reinterpret_cast<const double2 *>(p);
        const double2 q1 = *reinterpret_cast<const double2 *>(p + 2);
        o.c[0] = q0.x; o.c[1] = q0.y; o.c[2] = q1.x; o.c[3] = q1.y;
    }
    o.l = p[-1];
    o.r = p[4];
    return o;
}

template <typename T> __device__ __forceinline__ void load_cells4(const T *p, T (&c)[4]) {
    if constexpr (sizeof(T) == 4) {
        const float4 q = *reinterpret_cast<const float4 *>(p);
        c[0] = q.x; c[1] = q.y; c[2] = q.z; c[3] = q.w;
    } else {
        const double2 q0 = *reinterpret_cast<const double2 *>(p);
        const double2 q1 = *reinterpret_cast<const double2 *>(p + 2);
        c[0] = q0.x; c[1] = q0.y; c[2] = q1.x; c[3] = q1.y;
    }
}

template <typename TO> __device__ __forceinline__ void store4(TO *p, const Vec4<TO> &v, bool vec_ok,
                                                            int nvalid) {
    if (vec_ok && nvalid == 4) {
        if constexpr (sizeof(TO) == 4) {
            __stcs(reinterpret_cast<float4 *>(p), make_float4(v.v[0], v.v[1], v.v[2], v.v[3]));
        } else {
            __stcs(reinterpret_cast<double2 *>(p), make_double2(v.v[0], v.v[1]));
            __stcs(reinterpret_cast<double2 *>(p + 2), make_double2(v.v[2], v.v[3]));
        }
    } else {
#pragma unroll
        for (int i = 0; i < 4; ++i)
            if (i < nvalid) p[i] = v.v[i];
    }
}

template <typename TO> __device__ __forceinline__ void store4v(TO *p, const Vec4<TO> &v) {
    if constexpr (sizeof(TO) == 4) {
        __stcs(reinterpret_cast<float4 *>(p), make_float4(v.v[0], v.v[1], v.v[2], v.v[3]));
    } else {
        __stcs(reinterpret_cast<double2 *>(p), make_double2(v.v[0], v.v[1]));
        __stcs(reinterpret_cast<double2 *>(p + 2), make_double2(v.v[2], v.v[3]));
    }
}

// 4 cells into the shared-memory output staging (16-byte aligned: one st.shared.v4 for f32)
template <typename TO> __device__ __forceinline__ void store4_smem(TO *p, const Vec4<TO> &v) {
    if constexpr (sizeof(TO) == 4) {
        *reinterpret_cast<float4 *>(p) = make_float4(v.v[0], v.v[1], v.v[2], v.v[3]);
    } else {
        *reinterpret_cast<double2 *>(p) = make_double2(v.v[0], v.v[1]);
        *reinterpret_cast<double2 *>(p + 2) = make_double2(v.v[2], v.v[3]);
    }
}

// Operator concept (see surface_ops.cuh):
//   using in_t = float|double;  static constexpr int kOutputs;  using out_t;
//   struct Params;  __device__ Op(const Params&);
//   __device__ void step(const Row6<in_t>& row, Vec4<out_t> (&out)[kOutputs]);
//       -- consumes input row y and produces the outputs of row y-1 (valid once three
//          rows have been pushed).

struct StripGeom {
    int64_t H, W;
    int n_strips, n_segs, seg_rows;
};

template <typename Op> struct OutPtrs {
    typename Op::out_t *p[Op::kOutputs];
    int64_t pitch_elems;  // same for every output
};

// ----------------------------------------------------------------------------- TMA kernel
constexpr int kSubW = 208;  // cells per TMA box row (832 B for f32): 16-byte multiple, <= 256 elements

struct TileGeom {
    int64_t H, W;
    int n_tiles, n_segs, seg_rows;
};

// Source element type TS of the raster in HBM (== the operator's input type for the plain kernels;
// int16 / uint16 / int32 / float64 for direct ingestion, converted in registers with astype's
// rounding).  The halo is 32 bytes (8 cells of 4 bytes, 16 of 2, 4 of 8): with an aligned raster every
// box row then starts on a 32-byte L2 sector, and no sector is requested by two boxes.  With a 16-byte
// halo every float32 box row started 16 B into a sector; slope, hillshade and focal.mean each took 2-3 %
// longer on an H100 (DESIGN 4.1).  The pad must stay a multiple of 4 cells, so that a lane's 4 cells
// never straddle two boxes (kSubW is one too).
template <typename TS> struct SrcPad { static constexpr int value = 32 / (int)sizeof(TS); };

template <int WARPS, int PAD = kPad> struct TileShape {
    static constexpr int kTileW = kStripW * WARPS;                       // output columns per CTA tile
    static constexpr int kNSub = (kTileW + 2 * PAD + kSubW - 1) / kSubW;  // TMA boxes per stage
};

// 4 consecutive source cells -> operator input type
template <typename TI, typename TS> __device__ __forceinline__ void load_cells4_as(const TS *p, TI (&c)[4]) {
    if constexpr (sizeof(TS) == sizeof(TI) && !(TS(0.5) == TS(0))) {
        load_cells4<TI>(reinterpret_cast<const TI *>(p), c);   // same floating type
    } else if constexpr (sizeof(TS) == 2) {
        const uint2 q = *reinterpret_cast<const uint2 *>(p);
        TS e[4];
        memcpy(e, &q, 8);
#pragma unroll
        for (int i = 0; i < 4; ++i) c[i] = (TI)e[i];
    } else if constexpr (sizeof(TS) == 4) {
        const int4 q = *reinterpret_cast<const int4 *>(p);
        TS e[4];
        memcpy(e, &q, 16);
#pragma unroll
        for (int i = 0; i < 4; ++i) c[i] = (TI)e[i];
    } else {
        const double2 q0 = *reinterpret_cast<const double2 *>(p);
        const double2 q1 = *reinterpret_cast<const double2 *>(p + 2);
        c[0] = (TI)q0.x; c[1] = (TI)q0.y; c[2] = (TI)q1.x; c[3] = (TI)q1.y;
    }
}

// Shared-memory plan of one TMA-kernel instantiation: the input ring, then (bulk-store epilogue) kOutBufs
// staging buffers of ROWS x kTileW cells per output, then the mbarriers.  The bulk epilogue is used when
// CTAS such CTAs fit in an SM's 228 KB (1 KB of it reserved per CTA); otherwise lanes store from registers.
constexpr int kOutBufs = 2;

template <typename Op, int ROWS, int STAGES, int WARPS, int CTAS, typename TS = typename Op::in_t,
          int PAD = SrcPad<TS>::value>
struct TmaCfg {
    static constexpr int kPadS = PAD;
    static constexpr int kTileW = TileShape<WARPS, kPadS>::kTileW;
    static constexpr size_t kRingBytes = (size_t)STAGES * TileShape<WARPS, kPadS>::kNSub * ROWS * kSubW * sizeof(TS);
    static constexpr size_t kOutBufBytes = (size_t)ROWS * kTileW * Op::kOutputs * sizeof(typename Op::out_t);
    static constexpr size_t kBulkSmem = kRingBytes + kOutBufs * kOutBufBytes + (2 * STAGES + 2 * kOutBufs) * sizeof(uint64_t);
    static constexpr size_t kRegSmem = kRingBytes + 2 * STAGES * sizeof(uint64_t);
    static constexpr bool kBulk = kBulkSmem <= kSmemPerCtaMax && CTAS * (kBulkSmem + kSmemReservedPerCta) <= kSmemPerSm;
};

template <typename Op, int ROWS, int STAGES, int WARPS, typename TS, int PAD, bool BULK>
__global__ void __launch_bounds__((WARPS + 1 + (BULK ? 1 : 0)) * 32)
stencil3_tma_kernel(const __grid_constant__ CUtensorMap tmap,
                    const __grid_constant__ typename Op::Params prm,
                    const OutPtrs<Op> outs, const TileGeom g) {
    using TI = typename Op::in_t;   // what the operator consumes
    using T = TS;                   // what the ring holds
    using TO = typename Op::out_t;
    constexpr int kPadS = PAD;
    static_assert(PAD % kLaneCells == 0 && kSubW % kLaneCells == 0, "a lane's cells must lie in one box");
    constexpr bool kIntegral = (TS(0.5) == TS(0));   // integer cells: the TMA unit zero-fills, NaN comes from coordinates
    constexpr int kTileW = TileShape<WARPS, kPadS>::kTileW;
    constexpr int kNSub = TileShape<WARPS, kPadS>::kNSub;
    constexpr int kBoxElems = ROWS * kSubW;
    constexpr int kStageElems = kNSub * kBoxElems;
    constexpr uint32_t kStageBytes = kStageElems * sizeof(T);
    constexpr int kOutBufElems = BULK ? ROWS * kTileW * Op::kOutputs : 0;   // one staging buffer, [output][row][cell]
    static_assert((kBoxElems * sizeof(T)) % 128 == 0, "TMA destination must stay 128-byte aligned");

    extern __shared__ __align__(1024) unsigned char smem_raw[];
    T *ring = reinterpret_cast<T *>(smem_raw);
    TO *ostage = reinterpret_cast<TO *>(smem_raw + (size_t)STAGES * kStageBytes);
    uint64_t *full = reinterpret_cast<uint64_t *>(smem_raw + (size_t)STAGES * kStageBytes +
                                                  (size_t)kOutBufs * kOutBufElems * sizeof(TO));
    uint64_t *empty = full + STAGES;
    uint64_t *out_full = empty + STAGES;      // BULK only: WARPS arrivals, the staging buffer is written
    uint64_t *out_empty = out_full + kOutBufs; // BULK only: one arrival, the bulk copies have read it
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmap);
#pragma unroll
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], WARPS);
        }
        if constexpr (BULK) {
#pragma unroll
            for (int b = 0; b < kOutBufs; ++b) {
                mbar_init(&out_full[b], WARPS);
                mbar_init(&out_empty[b], 1);
            }
        }
        mbar_fence_init();
    }
    __syncthreads();

    const int64_t n_tasks = (int64_t)g.n_tiles * g.n_segs;

    if (BULK && warp == WARPS + 1) {
        // ---- store warp: one bulk copy per output row of the tile, in the consumers' (task, chunk) order
        if (lane == 0) {
            int ob = 0;
            uint32_t phase = 0;  // bit b = parity to wait for on out_full[b]
            for (int64_t task = blockIdx.x; task < n_tasks; task += gridDim.x) {
                const int seg = (int)(task / g.n_tiles), tile = (int)(task % g.n_tiles);
                const int64_t y0 = (int64_t)seg * g.seg_rows;
                const int seg_h = (int)(min(y0 + (int64_t)g.seg_rows, g.H) - y0);
                const int n_chunks = (seg_h + 2 + ROWS - 1) / ROWS;
                const int64_t x0 = (int64_t)tile * kTileW;
                // W % 4 == 0 on this path: every row copy is a multiple of 16 bytes
                const uint32_t bytes = (uint32_t)(min((int64_t)kTileW, g.W - x0) * (int64_t)sizeof(TO));
                for (int c = 0; c < n_chunks; ++c) {
                    mbar_wait(&out_full[ob], (phase >> ob) & 1u);
                    phase ^= (1u << ob);
                    const TO *src = ostage + ob * kOutBufElems;
                    const int rel = c * ROWS - 2;  // output row (relative to y0) of the chunk's first row
#pragma unroll
                    for (int r = 0; r < ROWS; ++r) {
                        if ((unsigned)(rel + r) >= (unsigned)seg_h) continue;  // lead-in rows / past the raster
                        const int64_t off = (y0 + rel + r) * outs.pitch_elems + x0;
#pragma unroll
                        for (int k = 0; k < Op::kOutputs; ++k)
                            if (Op::kOutputs == 1 || outs.p[k] != nullptr)
                                bulk_store(outs.p[k] + off, src + (k * ROWS + r) * kTileW, bytes);
                    }
                    bulk_commit();
                    bulk_wait_read_all();  // the staging buffer may be rewritten ...
                    mbar_arrive(&out_empty[ob]);  // ... while its global writes drain
                    ob = (ob + 1 == kOutBufs) ? 0 : ob + 1;
                }
            }
            bulk_wait_read_all();
        }
        return;
    }

    if (warp == WARPS) {
        // ---- producer: walks the same (task, chunk) sequence as the consumers, STAGES ahead
        if (lane == 0) {
            int stage = 0;
            // Input lines are kept in L2 with evict_last priority, so the L2 evicts (writes back) the
            // output lines first.  On an H100 this is 1.6 % faster than no hint for every 3x3 operator;
            // evict_first on the loads is 3.5 % slower (DESIGN 4.1).
            const uint64_t keep = l2_policy_evict_last();
            uint32_t phase = 0;  // bit s = parity of the `empty` phase stage s was last refilled under
            for (int64_t task = blockIdx.x; task < n_tasks; task += gridDim.x) {
                const int seg = (int)(task / g.n_tiles), tile = (int)(task % g.n_tiles);
                const int64_t y0 = (int64_t)seg * g.seg_rows;
                const int64_t y1 = min(y0 + (int64_t)g.seg_rows, g.H);
                const int n_chunks = ((int)(y1 - y0) + 2 + ROWS - 1) / ROWS;  // input rows y0-1 .. y1
                const int bx = tile * kTileW - kPadS, by = (int)y0 - 1;
                for (int c = 0; c < n_chunks; ++c) {
                    // a fresh barrier passes a wait on parity 1: the first lap never blocks
                    mbar_wait(&empty[stage], ((phase >> stage) & 1u) ^ 1u);
                    phase ^= (1u << stage);
                    mbar_arrive_expect_tx(&full[stage], kStageBytes);
                    T *dst = ring + stage * kStageElems;
#pragma unroll
                    for (int b = 0; b < kNSub; ++b)
                        tma_load_2d_hint(dst + b * kBoxElems, &tmap, &full[stage], bx + b * kSubW, by + c * ROWS,
                                         keep);
                    stage = (stage + 1 == STAGES) ? 0 : stage + 1;
                }
            }
        }
        return;
    }

    // ---- consumers.  Column cc of the stage (0 = first halo cell) lives in box cc / kSubW.
    const int cc = kPadS + kStripW * warp + kLaneCells * lane;
    const int off_c = (cc / kSubW) * kBoxElems + cc % kSubW;
    const int off_l = ((cc - 1) / kSubW) * kBoxElems + (cc - 1) % kSubW;
    const int off_r = ((cc + kLaneCells) / kSubW) * kBoxElems + (cc + kLaneCells) % kSubW;
    int stage = 0;
    uint32_t phase = 0;  // bit s = parity to wait for on full[s]
    int ob = 0;
    uint32_t ophase = 0;  // BULK: bit b = parity of the out_empty phase buffer b was last written under
    TO *const my_stage = ostage + kStripW * warp + kLaneCells * lane;   // BULK: this lane's cells, buffer 0, row 0
    for (int64_t task = blockIdx.x; task < n_tasks; task += gridDim.x) {
        const int seg = (int)(task / g.n_tiles), tile = (int)(task % g.n_tiles);
        const int64_t y0 = (int64_t)seg * g.seg_rows;
        const int64_t y1 = min(y0 + (int64_t)g.seg_rows, g.H);
        const int seg_h = (int)(y1 - y0);
        const int n_chunks = (seg_h + 2 + ROWS - 1) / ROWS;

        Op op(prm);
        const int64_t xl = (int64_t)tile * kTileW + kStripW * warp + kLaneCells * lane;
        const bool lane_ok = xl < g.W;  // W % 4 == 0 on this path: a lane is all-in or all-out
        const bool left_oob = xl == 0, right_oob = xl + 4 >= g.W;   // integer sources only
        // register stores: output pointers one row above the first emitted row (y0 - 2), advanced before every store
        TO *optr[Op::kOutputs];
        if constexpr (!BULK) {
#pragma unroll
            for (int k = 0; k < Op::kOutputs; ++k) optr[k] = outs.p[k] + (y0 - 3) * outs.pitch_elems + xl;
        }

        for (int c = 0; c < n_chunks; ++c) {
            mbar_wait(&full[stage], (phase >> stage) & 1u);
            phase ^= (1u << stage);
            TO *ost = my_stage + ob * kOutBufElems;
            if constexpr (BULK) {
                // a fresh barrier passes a wait on parity 1: the first lap never blocks
                mbar_wait(&out_empty[ob], ((ophase >> ob) & 1u) ^ 1u);
                ophase ^= (1u << ob);
            }
            const T *buf = ring + stage * kStageElems;
            const int rel = c * ROWS - 2;  // output row (relative to y0) of the stage's first row
            const int64_t ybase = y0 - 1 + (int64_t)c * ROWS;
            // Straight-line over the ROWS rows of the stage (no branch around the operator state
            // update, so the rolling registers are renamed, not moved).  Rows whose output row
            // falls outside [y0, y1) -- the two lead-in rows and the tail of the last chunk --
            // still update the state; only their store is predicated off.
#pragma unroll
            for (int r = 0; r < ROWS; ++r) {
                Row6<TI> row;
                load_cells4_as<TI, TS>(buf + off_c + r * kSubW, row.c);
                row.l = (TI)buf[off_l + r * kSubW];
                row.r = (TI)buf[off_r + r * kSubW];
                if constexpr (kIntegral) {
                    const int64_t y = ybase + r;
                    const bool row_oob = (y < 0) || (y >= g.H);
                    if (row_oob || left_oob) row.l = nan_of<TI>();
                    if (row_oob || right_oob) row.r = nan_of<TI>();
                    if (row_oob || !lane_ok) row.c[0] = row.c[1] = row.c[2] = row.c[3] = nan_of<TI>();
                }
                Vec4<TO> o[Op::kOutputs];
                op.step(row, o);
                if constexpr (BULK) {
                    // every row goes to the staging buffer; the store warp copies only rows in [y0, y1)
                    // and only the columns left of W
#pragma unroll
                    for (int k = 0; k < Op::kOutputs; ++k)
                        if (Op::kOutputs == 1 || outs.p[k] != nullptr) store4_smem<TO>(ost + (k * ROWS + r) * kTileW, o[k]);
                } else {
                    const bool st = lane_ok && (unsigned)(rel + r) < (unsigned)seg_h;
#pragma unroll
                    for (int k = 0; k < Op::kOutputs; ++k) {
                        optr[k] += outs.pitch_elems;
                        if (st && (Op::kOutputs == 1 || outs.p[k] != nullptr)) store4v<TO>(optr[k], o[k]);
                    }
                }
            }
            if constexpr (BULK) fence_proxy_async_smem();  // this lane's staging writes, visible to the bulk copies
            __syncwarp();  // every lane is done reading this stage (and writing its staging cells)
            if (lane == 0) {
                mbar_arrive(&empty[stage]);
                if constexpr (BULK) mbar_arrive(&out_full[ob]);
            }
            stage = (stage + 1 == STAGES) ? 0 : stage + 1;
            if constexpr (BULK) ob = (ob + 1 == kOutBufs) ? 0 : ob + 1;
        }
    }
}

// ----------------------------------------------------------------------------- cp.async kernel
// Same warp-strip pipeline for rasters TMA cannot describe (width not a multiple of 4 cells, base
// or pitch not 16-byte aligned): the per-warp ring is filled with 4-/8-byte cp.async copies
// (coalesced: lane i copies cells i, i+32, ... of the box row; out-of-raster cells are written
// as NaN with plain stores), completion is tracked with cp.async groups instead of mbarriers.
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
template <typename T> __device__ __forceinline__ void cp_async_elem(T *dst, const T *src) {
    if constexpr (sizeof(T) == 4)
        asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
    else
        asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}

template <typename Op, int ROWS, int STAGES>
__global__ void __launch_bounds__(kWarpsPerCta * 32)
stencil3_cpasync_kernel(const typename Op::in_t *__restrict__ in, int64_t in_pitch_elems,
                        const __grid_constant__ typename Op::Params prm, const OutPtrs<Op> outs,
                        const StripGeom g, int vec_ok) {
    using T = typename Op::in_t;
    using TO = typename Op::out_t;
    constexpr int kStageElems = ROWS * kBoxW;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    T *ring = reinterpret_cast<T *>(smem_raw) + (size_t)warp * STAGES * kStageElems;

    const int64_t n_tasks = (int64_t)g.n_strips * g.n_segs;
    const int64_t total_warps = (int64_t)gridDim.x * kWarpsPerCta;
    for (int64_t task = (int64_t)blockIdx.x * kWarpsPerCta + warp; task < n_tasks; task += total_warps) {
        const int seg = (int)(task / g.n_strips), strip = (int)(task % g.n_strips);
        const int64_t x0 = (int64_t)strip * kStripW;
        const int64_t y0 = (int64_t)seg * g.seg_rows;
        const int64_t y1 = min(y0 + (int64_t)g.seg_rows, g.H);
        const int rows_in = (int)(y1 - y0) + 2;
        const int n_chunks = (rows_in + ROWS - 1) / ROWS;
        const int64_t bx = x0 - kPad, by = y0 - 1;

        auto fill = [&](int c) {  // chunk c -> stage c % STAGES
            if (c < n_chunks) {
                T *dst = ring + (c % STAGES) * kStageElems;
#pragma unroll
                for (int r = 0; r < ROWS; ++r) {
                    const int64_t y = by + (int64_t)c * ROWS + r;
                    const bool yin = (y >= 0) && (y < g.H);
                    const T *rp = in + (yin ? y : 0) * in_pitch_elems;
#pragma unroll
                    for (int j0 = 0; j0 < kBoxW; j0 += 32) {
                        const int j = j0 + lane;
                        const int64_t x = bx + j;
                        if (j < kBoxW) {
                            if (yin && x >= 0 && x < g.W) cp_async_elem<T>(dst + r * kBoxW + j, rp + x);
                            else dst[r * kBoxW + j] = nan_of<T>();
                        }
                    }
                }
            }
            cp_async_commit();  // one group per chunk slot, possibly empty
        };

#pragma unroll
        for (int c = 0; c < STAGES - 1; ++c) fill(c);

        Op op(prm);
        const int64_t xl = x0 + kLaneCells * lane;
        const int nvalid = (int)max((int64_t)0, min((int64_t)4, g.W - xl));
        const int seg_h = (int)(y1 - y0);
        const T *lane_smem = ring + kPad + kLaneCells * lane;
        TO *optr[Op::kOutputs];
#pragma unroll
        for (int k = 0; k < Op::kOutputs; ++k) optr[k] = outs.p[k] + (y0 - 3) * outs.pitch_elems + xl;

        for (int c = 0; c < n_chunks; ++c) {
            fill(c + STAGES - 1);
            cp_async_wait<STAGES - 1>();  // this lane's copies of chunk c have landed ...
            __syncwarp();                 // ... and so have the other lanes'
            const T *buf = lane_smem + (c % STAGES) * kStageElems;
            const int rel = c * ROWS - 2;
#pragma unroll
            for (int r = 0; r < ROWS; ++r) {
                const Row6<T> row = load_row_smem<T>(buf + r * kBoxW);
                Vec4<TO> o[Op::kOutputs];
                op.step(row, o);
                const bool st = nvalid > 0 && (unsigned)(rel + r) < (unsigned)seg_h;
#pragma unroll
                for (int k = 0; k < Op::kOutputs; ++k) {
                    optr[k] += outs.pitch_elems;
                    if (st && (Op::kOutputs == 1 || outs.p[k] != nullptr))
                        store4<TO>(optr[k], o[k], vec_ok != 0, nvalid);
                }
            }
            __syncwarp();  // every lane is done with this stage before it is refilled
        }
        cp_async_wait<0>();
    }
}

// ----------------------------------------------------------------------------- host launcher
// Row segments.  Tasks (tiles x segments) are dealt round-robin to `resident` persistent CTAs, so a kernel
// lasts ceil(tasks / resident) task-times ("waves"): one task too many costs a whole extra wave (1188 tasks on
// 1184 task slots ran 9 waves instead of 8.03: the round-2 fused suite lost 11 % to that).  Pick the
// segment height that minimises waves x (rows + lead-in rows a task streams), among heights of at least
// `min_rows` with (rows + lead) a multiple of `quantum` (so the last chunk of a segment is full); among
// heights within 1 % of the best prefer ~`want` waves (short tasks even out the partly filled last tile).
// make_tile_geom asks for ~2 waves: at 32768^2 on an H100, long segments (fewer lead-in rows, fewer task
// switches) were 0.4 % faster than ~8 waves for the 3x3 operators.
inline int64_t pick_seg_rows(int64_t H, int64_t n_tiles, int64_t resident, int64_t min_rows, int64_t lead,
                             int64_t quantum, int64_t want) {
    if (H <= 0) return 1;
    if (resident < 1) resident = 1;
    if (min_rows > H) min_rows = H;
    if (min_rows < 1) min_rows = 1;
    int64_t cmax = H / min_rows;
    const int64_t ccap = (resident * 4 * want) / (n_tiles > 0 ? n_tiles : 1) + 2;
    if (cmax > ccap) cmax = ccap;
    if (cmax < 1) cmax = 1;
    double best = 0.0;
    for (int pass = 0; pass < 2; ++pass) {
        int64_t pick = 0, pick_d = 0;
        for (int64_t c = 1; c <= cmax; ++c) {
            int64_t rows = (H + c - 1) / c;
            if (rows < min_rows) rows = min_rows;
            rows = ((rows + lead + quantum - 1) / quantum) * quantum - lead;
            if (rows < 1) rows = 1;
            const int64_t segs = (H + rows - 1) / rows;
            const int64_t waves = (segs * n_tiles + resident - 1) / resident;
            const double cost = (double)waves * (double)(rows + lead);
            if (pass == 0) {
                if (best == 0.0 || cost < best) best = cost;
            } else if (cost <= best * 1.01) {
                const int64_t d = waves > want ? waves - want : want - waves;
                if (pick == 0 || d < pick_d) { pick = rows; pick_d = d; }
            }
        }
        if (pass == 1) return pick > 0 ? pick : H;
    }
    return H;
}

inline TileGeom make_tile_geom(int64_t H, int64_t W, int tile_w, int rows, int64_t resident_ctas) {
    TileGeom g;
    g.H = H;
    g.W = W;
    g.n_tiles = (int)((W + tile_w - 1) / tile_w);
    const int64_t seg_rows = pick_seg_rows(H, g.n_tiles, resident_ctas, 32, 2, rows, 2);
    g.seg_rows = (int)seg_rows;
    g.n_segs = (int)((H + seg_rows - 1) / seg_rows);
    return g;
}

// ROWS x STAGES = the TMA ring of the CTA-wide pipeline, WARPS consumer warps per CTA, CTAS CTAs per
// SM: tuned per operator (surface.cu, scripts/tune/tune5.cu).  `kind` is what LaunchInfo::kind reports.
// BULK defaults to the bulk-store epilogue wherever its staging fits; the tuning harness also times the
// register-store epilogue, and other halo widths PAD.
template <typename Op, int ROWS, int STAGES, int WARPS, int CTAS, typename TS = typename Op::in_t,
          int PAD = SrcPad<TS>::value, bool BULK = TmaCfg<Op, ROWS, STAGES, WARPS, CTAS, TS, PAD>::kBulk>
int launch_tma(const CUtensorMap &tmap, const typename Op::Params &prm, const OutPtrs<Op> &outs, int64_t H,
               int64_t W, cudaStream_t stream, LaunchKind kind) {
    using Cfg = TmaCfg<Op, ROWS, STAGES, WARPS, CTAS, TS, PAD>;
    static_assert(!BULK || Cfg::kBulk, "the bulk-store staging does not fit next to this ring");
    constexpr size_t smem = BULK ? Cfg::kBulkSmem : Cfg::kRegSmem;
    constexpr int threads = (WARPS + 1 + (BULK ? 1 : 0)) * 32;  // consumers, producer[, store warp]
    auto kern = stencil3_tma_kernel<Op, ROWS, STAGES, WARPS, TS, PAD, BULK>;
    // persistent grid: CTAS per SM (or what fits), never more CTAs than tasks
    int64_t resident;
    if (const int rc = resident_ctas(kern, threads, smem, CTAS, &resident)) return rc;
    const TileGeom g = make_tile_geom(H, W, Cfg::kTileW, ROWS, resident);
    const int64_t n_tasks = (int64_t)g.n_tiles * g.n_segs;
    return launch(kern, resident < n_tasks ? resident : n_tasks, threads, smem, stream, kind, tmap, prm, outs, g);
}

// The TMA strip kernel takes a raster when W % 4 == 0 (a lane's 4 cells are all inside or all outside), the
// output rows are 16-byte aligned (bulk copies and float4 stores) and TMA can describe the input; then `map`
// holds the input's tensor map.
template <typename TS>
bool strip_tma_map(CUtensorMap *map, const TS *in, int64_t in_pitch_bytes, int64_t H, int64_t W, int rows,
                   bool out_aligned) {
    return out_aligned && W % 4 == 0 && make_tensor_map_2d(map, in, in_pitch_bytes, H, W, dtype_of<TS>(), kSubW, rows);
}

constexpr int kFallbackRows = 4, kFallbackStages = 4;  // cp.async ring (per warp)

// Checks the arguments, then runs the TMA kernel when strip_tma_map takes the raster, else the cp.async kernel.
// TS is the cell type in HBM: for TS != Op::in_t (int16 / uint16 / int32 / float64 cells converted in registers)
// only the TMA kernel exists, and other layouts return XRS_EUNSUPPORTED.
template <typename Op, int ROWS, int STAGES, int WARPS, int CTAS, typename TS = typename Op::in_t>
int launch_stencil3(const TS *in, int64_t in_pitch_bytes, const typename Op::Params &prm,
                    typename Op::out_t *const *out_ptrs, int64_t out_pitch_bytes, int64_t H, int64_t W,
                    cudaStream_t stream) {
    using T = typename Op::in_t;
    using TO = typename Op::out_t;
    constexpr bool kConvert = !std::is_same<TS, T>::value;
    if (H <= 0 || W <= 0) return XRS_OK;  // empty raster: nothing to do
    XRS_TRY(check_cells_arg(in, dtype_of<TS>(), kRasterCells, in_pitch_bytes, W));
    XRS_TRY(check_out_pitch(out_pitch_bytes, sizeof(TO), W));
    XRS_REQUIRE(H < (1LL << 31) - 8 && W < (1LL << 31) - 4096, "raster dimension too large");

    OutPtrs<Op> outs;
    bool any = false, out_vec_ok = (out_pitch_bytes % 16 == 0);
    for (int k = 0; k < Op::kOutputs; ++k) {
        outs.p[k] = out_ptrs[k];
        if (out_ptrs[k]) {
            any = true;
            XRS_REQUIRE((const void *)out_ptrs[k] != (const void *)in, "in and out must not alias");
            if (reinterpret_cast<uintptr_t>(out_ptrs[k]) % 16 != 0) out_vec_ok = false;
        }
    }
    XRS_REQUIRE(any, "no output pointer given");
    outs.pitch_elems = out_pitch_bytes / (int64_t)sizeof(TO);

    CUtensorMap tmap;
    if (strip_tma_map(&tmap, in, in_pitch_bytes, H, W, ROWS, out_vec_ok))
        return launch_tma<Op, ROWS, STAGES, WARPS, CTAS, TS>(tmap, prm, outs, H, W, stream,
                                                             kConvert ? kIngestTma : kStripTma);
    if constexpr (kConvert) {
        set_error("raster layout not supported by the direct-ingest path (needs 16-byte aligned rows, W %% 4 == 0)");
        return XRS_EUNSUPPORTED;
    } else {  // rasters TMA cannot describe: the per-warp cp.async ring
        constexpr int FR = sizeof(T) == 8 ? 2 : kFallbackRows, FS = kFallbackStages;
        StripGeom g;
        g.H = H;
        g.W = W;
        g.n_strips = (int)((W + kStripW - 1) / kStripW);
        const int64_t resident_warps = (int64_t)sm_count() * 2 * kWarpsPerCta;
        int64_t want_segs = (resident_warps * 8 + g.n_strips - 1) / g.n_strips;
        int64_t seg_rows = (H + want_segs - 1) / (want_segs > 0 ? want_segs : 1);
        if (seg_rows < 64) seg_rows = 64;
        if (seg_rows > H) seg_rows = H;
        seg_rows = ((seg_rows + 2 + FR - 1) / FR) * FR - 2;
        if (seg_rows < 1) seg_rows = 1;
        g.seg_rows = (int)seg_rows;
        g.n_segs = (int)((H + seg_rows - 1) / seg_rows);
        const int64_t n_tasks = (int64_t)g.n_strips * g.n_segs;
        const int64_t ctas_needed = (n_tasks + kWarpsPerCta - 1) / kWarpsPerCta;
        constexpr size_t smem = (size_t)kWarpsPerCta * FS * FR * kBoxW * sizeof(T);
        auto kern = stencil3_cpasync_kernel<Op, FR, FS>;
        int64_t resident;
        if (const int rc = resident_ctas(kern, kWarpsPerCta * 32, smem, 2, &resident)) return rc;
        return launch(kern, resident < ctas_needed ? resident : ctas_needed, kWarpsPerCta * 32, smem, stream,
                      kStripCpAsync, in, in_pitch_bytes / (int64_t)sizeof(T), prm, outs, g, out_vec_ok ? 1 : 0);
    }
}

}  // namespace xrs

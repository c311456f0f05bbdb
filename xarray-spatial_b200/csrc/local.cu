// local.cu -- the reference's local.py (cell_stats, the frequencies, the positions, popularity, rank, combine) over
// K layers, with the per-cell rule of local_rule.cuh.
//
// xrs_local_cells: one grid-stride kernel; each thread reads its cell from the K layers (typed loads, widened in
// registers) and writes the rule's result.  A stack of one cell type gets a kernel that reads that type directly;
// a mixed stack switches on each layer's code.  The op is a template argument, so each kernel holds one rule.
// xrs_local_combine: phase 0 inserts every non-NaN cell's index into an open-addressing table keyed by its tuple
// (atomicMin keeps the first occurrence); the caller numbers the occupied slots by first index and stores -1 - id
// in each; phase 1 looks every cell up again and writes its id (DESIGN.md section 4.13).
#include "common.cuh"
#include "local_rule.cuh"

namespace xrs {
namespace {

using namespace lc;

constexpr int kThreads = 256;
constexpr unsigned long long kEmpty = 0x7fffffffffffffffull;

struct Layer {
    const char *base;
    int64_t pitch;
    int64_t dtype;
};

template <typename T> __device__ __forceinline__ Val read_cell(const char *base, int64_t pitch, int64_t r, int64_t c) {
    return load(__ldg(reinterpret_cast<const T *>(base + r * pitch) + c));
}
template <> __device__ __forceinline__ Val read_cell<bool>(const char *base, int64_t pitch, int64_t r, int64_t c) {
    return ival(__ldg(reinterpret_cast<const unsigned char *>(base + r * pitch) + c) != 0, kBool);
}

__device__ Val read_any(const Layer &l, int64_t r, int64_t c) {
    switch (l.dtype) {
        case XRS_F32: return read_cell<float>(l.base, l.pitch, r, c);
        case XRS_F64: return read_cell<double>(l.base, l.pitch, r, c);
        case XRS_I32: return read_cell<int32_t>(l.base, l.pitch, r, c);
        case XRS_I64: return read_cell<long long>(l.base, l.pitch, r, c);
        case XRS_I16: return read_cell<int16_t>(l.base, l.pitch, r, c);
        case XRS_U16: return read_cell<uint16_t>(l.base, l.pitch, r, c);
        case XRS_I8: return read_cell<int8_t>(l.base, l.pitch, r, c);
        case XRS_U8: return read_cell<uint8_t>(l.base, l.pitch, r, c);
        case XRS_U32: return read_cell<uint32_t>(l.base, l.pitch, r, c);
        case XRS_U64: return read_cell<long long>(l.base, l.pitch, r, c);   // cells below 2**63
        default: return read_cell<bool>(l.base, l.pitch, r, c);
    }
}

// The first kSmemLayers descriptors are staged in shared memory by each CTA; deeper stacks read the rest from
// global memory.
constexpr int kSmemLayers = 512;

struct Layers {
    const Layer *smem, *global;
    __device__ Layer operator[](int64_t j) const { return j < kSmemLayers ? smem[j] : global[j]; }
};

__device__ Layers stage_layers(const Layer *layers, int64_t K) {
    extern __shared__ Layer staged[];
    for (int64_t j = threadIdx.x; j < K && j < kSmemLayers; j += blockDim.x) staged[j] = layers[j];
    __syncthreads();
    return Layers{staged, layers};
}

size_t stage_bytes(int64_t K) { return (size_t)(K < kSmemLayers ? K : kSmemLayers) * sizeof(Layer); }

// T: the stack's one cell type, or void for a mixed stack
template <typename T> struct Reader {
    Layers layers;
    int64_t r, c;
    __device__ Val operator()(int64_t j) const {
        const Layer l = layers[j];
        if constexpr (std::is_void_v<T>) return read_any(l, r, c);
        else return read_cell<T>(l.base, l.pitch, r, c);
    }
};

// The stack's array kind: fixed by the cell type of a one-type stack, so its kernel holds only that branch.
template <typename T> __device__ __forceinline__ int stack_kind(int ak) {
    if constexpr (std::is_void_v<T>) return ak;
    else if constexpr (std::is_same_v<T, bool>) return kBool;
    else if constexpr (std::is_floating_point_v<T>) return kFloat;
    else return kInt;
}

__device__ __forceinline__ void or_flags(unsigned *flags, unsigned f) {
    f = __reduce_or_sync(0xffffffffu, f);
    if (f && (threadIdx.x & 31) == 0) atomicOr(flags, f);
}

template <int OP, typename T>
__global__ void __launch_bounds__(kThreads) local_cells_kernel(const Layer *layers, int64_t K, int64_t H, int64_t W,
                                                              int ak, Layer ref, int ref_f16, int64_t *out,
                                                              int64_t out_pitch, uint8_t *kinds,
                                                              int64_t kinds_pitch, unsigned *flags) {
    const Layers l = stage_layers(layers, K);
    unsigned f = 0;
    const int64_t n = H * W;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = k / W, c = k - r * W;
        Ref rf{};
        if constexpr ((OP >= kLesser && OP <= kGreater) || OP >= kPopularity)
            rf = make_ref(read_any(ref, r, c), (int)ref.dtype, ref_f16 != 0);
        const Result res = cell(OP, K, stack_kind<T>(ak), Reader<T>{l, r, c}, rf);
        reinterpret_cast<int64_t *>(reinterpret_cast<char *>(out) + r * out_pitch)[c] = res.bits;
        if constexpr (OP >= kPopularity) kinds[r * kinds_pitch + c] = (uint8_t)res.kind;
        f |= res.flags;
    }
    or_flags(flags, f);
}

template <int OP> int launch_cells(int uniform, const Layer *layers, int64_t K, int64_t H, int64_t W, int ak,
                                   Layer ref, int ref_f16, int64_t *out, int64_t out_pitch, uint8_t *kinds,
                                   int64_t kinds_pitch, unsigned *flags, cudaStream_t s) {
    const int64_t grid = stride_grid(H * W);
    auto go = [&](auto t) -> int {
        using T = decltype(t);
        local_cells_kernel<OP, T><<<(unsigned)grid, kThreads, stage_bytes(K), s>>>(
            layers, K, H, W, ak, ref, ref_f16, out, out_pitch, kinds, kinds_pitch, flags);
        XRS_CUDA(cudaGetLastError());
        return XRS_OK;
    };
    if (uniform < 0) {
        local_cells_kernel<OP, void><<<(unsigned)grid, kThreads, stage_bytes(K), s>>>(
            layers, K, H, W, ak, ref, ref_f16, out, out_pitch, kinds, kinds_pitch, flags);
        XRS_CUDA(cudaGetLastError());
        return XRS_OK;
    }
    if (uniform == XRS_U64) return go((long long)0);   // cells below 2**63
    return with_cell_type(kZonalCells, uniform, go);
}

using CellsLauncher = int (*)(int, const Layer *, int64_t, int64_t, int64_t, int, Layer, int, int64_t *, int64_t,
                              uint8_t *, int64_t, unsigned *, cudaStream_t);
constexpr CellsLauncher kCellsLaunchers[kNumOps] = {
    launch_cells<0>, launch_cells<1>, launch_cells<2>, launch_cells<3>, launch_cells<4>,  launch_cells<5>,
    launch_cells<6>, launch_cells<7>, launch_cells<8>, launch_cells<9>, launch_cells<10>, launch_cells<11>,
    launch_cells<12>};

// ---------------------------------------------------------------------------------------------- combine
using AnyReader = Reader<void>;

__device__ __forceinline__ bool tuple_nan(int64_t K, const AnyReader &x) {
    for (int64_t j = 0; j < K; ++j)
        if (is_nan(x(j))) return true;
    return false;
}

__global__ void __launch_bounds__(kThreads) combine_fill(unsigned long long *table, int64_t slots) {
    for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < slots; s += (int64_t)gridDim.x * blockDim.x)
        table[s] = kEmpty;
}

__global__ void __launch_bounds__(kThreads) combine_insert(const Layer *layers, int64_t K, int64_t H, int64_t W,
                                                          unsigned long long *table, uint64_t mask,
                                                          unsigned *flags) {
    const Layers l = stage_layers(layers, K);
    unsigned f = 0;
    const int64_t n = H * W;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
        const AnyReader x{l, k / W, k % W};
        if (tuple_nan(K, x)) {
            f |= kFlagNan;
            continue;
        }
        for (uint64_t s = tuple_hash(K, x) & mask;; s = (s + 1) & mask) {
            unsigned long long cur = __ldcg(table + s);
            if (cur == kEmpty) {
                cur = atomicCAS(table + s, kEmpty, (unsigned long long)k);
                if (cur == kEmpty) break;
            }
            const AnyReader y{l, (int64_t)cur / W, (int64_t)cur % W};
            if (tuple_equal(K, x, y)) {
                atomicMin(table + s, (unsigned long long)k);
                break;
            }
        }
    }
    or_flags(flags, f);
}

// table[s] = -1 - id for every occupied slot; reps[id] is the id's first cell
__global__ void __launch_bounds__(kThreads) combine_label(const Layer *layers, int64_t K, int64_t H, int64_t W,
                                                         const long long *table, uint64_t mask,
                                                         const long long *reps, int64_t *out, int64_t out_pitch) {
    const Layers l = stage_layers(layers, K);
    const int64_t n = H * W;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = k / W, c = k - r * W;
        const AnyReader x{l, r, c};
        int64_t id = -1;
        if (!tuple_nan(K, x)) {
            for (uint64_t s = tuple_hash(K, x) & mask;; s = (s + 1) & mask) {
                const int64_t u = -1 - __ldg(table + s);
                const int64_t rep = __ldg(reps + u);
                if (tuple_equal(K, x, AnyReader{l, rep / W, rep % W})) {
                    id = u + 1;
                    break;
                }
            }
        }
        reinterpret_cast<int64_t *>(reinterpret_cast<char *>(out) + r * out_pitch)[c] = id;
    }
}

// Table slots: a power of two, at least twice the cells.
int64_t combine_slots(int64_t H, int64_t W) {
    int64_t c = 2;
    while (c < 2 * H * W) c <<= 1;
    return c;
}

// Checks the K host layer descriptors {pointer, pitch, dtype}, copies them to dev; *uniform = their one dtype,
// or -1.
int take_layers(const int64_t *host, int64_t K, void *dev, int64_t W, cudaStream_t s, int *uniform) {
    XRS_REQUIRE(host != nullptr && dev != nullptr, "NULL layer descriptors");
    XRS_REQUIRE(K >= 1, "no layers");
    *uniform = (int)host[2];
    for (int64_t j = 0; j < K; ++j) {
        XRS_TRY(check_cells_arg((const void *)host[3 * j], (int)host[3 * j + 2], kZonalCells, host[3 * j + 1], W));
        if (host[3 * j + 2] != *uniform) *uniform = -1;
    }
    XRS_CUDA(cudaMemcpyAsync(dev, host, (size_t)K * sizeof(Layer), cudaMemcpyHostToDevice, s));
    return XRS_OK;
}

}  // namespace
}  // namespace xrs

using namespace xrs;

extern "C" int xrs_local_cells(const int64_t *layers, int64_t K, void *layers_dev, int64_t H, int64_t W, int op,
                               int ak, const void *ref, int64_t ref_pitch, int ref_dtype, int ref_f16, int64_t *out,
                               int64_t out_pitch, uint8_t *kinds, int64_t kinds_pitch, unsigned *flags,
                               void *stream) {
    XRS_REQUIRE(H >= 0 && W >= 0, "negative raster size");
    XRS_REQUIRE(op >= 0 && op < lc::kNumOps, "unknown local op");
    XRS_REQUIRE(ak >= lc::kFloat && ak <= lc::kBool, "unknown array kind");
    XRS_REQUIRE(out != nullptr && flags != nullptr, "NULL output");
    XRS_TRY(check_out_pitch(out_pitch, 8, W));
    const bool takes_ref = (op >= lc::kLesser && op <= lc::kGreater) || op >= lc::kPopularity;
    if (takes_ref) {
        XRS_TRY(check_cells_arg(ref, ref_dtype, kZonalCells, ref_pitch, W));
        XRS_REQUIRE(!ref_f16 || ref_dtype == XRS_F32, "float16 refs are carried as float32");
    }
    if (op >= lc::kPopularity) {
        XRS_REQUIRE(kinds != nullptr, "NULL kinds");
        XRS_REQUIRE(kinds_pitch >= W, "bad kinds pitch");
    }
    if (H == 0 || W == 0) return XRS_OK;
    const cudaStream_t s = (cudaStream_t)stream;
    int uniform;
    XRS_TRY(take_layers(layers, K, layers_dev, W, s, &uniform));
    const Layer rl{(const char *)ref, ref_pitch, ref_dtype};
    return kCellsLaunchers[op](uniform, (const Layer *)layers_dev, K, H, W, ak, rl, ref_f16, out, out_pitch, kinds,
                               kinds_pitch, flags, s);
}

extern "C" int xrs_local_combine_scratch_bytes(int64_t H, int64_t W, int64_t *bytes) {
    XRS_REQUIRE(H >= 0 && W >= 0, "negative raster size");
    XRS_REQUIRE(bytes != nullptr, "NULL bytes");
    *bytes = 8 * combine_slots(H, W);
    return XRS_OK;
}

extern "C" int xrs_local_combine(const int64_t *layers, int64_t K, void *layers_dev, int64_t H, int64_t W, int phase,
                                 void *scratch, int64_t scratch_bytes, const int64_t *reps, int64_t *out,
                                 int64_t out_pitch, unsigned *flags, void *stream) {
    XRS_REQUIRE(H >= 0 && W >= 0, "negative raster size");
    XRS_REQUIRE(phase == 0 || phase == 1, "unknown combine phase");
    XRS_REQUIRE(out != nullptr && flags != nullptr, "NULL output");
    XRS_TRY(check_out_pitch(out_pitch, 8, W));
    const int64_t slots = combine_slots(H, W);
    XRS_TRY(check_scratch(scratch, scratch_bytes, 8 * slots, "xrs_local_combine_scratch_bytes"));
    XRS_REQUIRE(phase == 0 || reps != nullptr, "NULL reps");
    if (H == 0 || W == 0) return XRS_OK;
    const cudaStream_t s = (cudaStream_t)stream;
    int uniform;
    XRS_TRY(take_layers(layers, K, layers_dev, W, s, &uniform));
    const Layer *l = (const Layer *)layers_dev;
    const int64_t grid = stride_grid(H * W);
    auto *table = (unsigned long long *)scratch;
    if (phase == 0) {
        combine_fill<<<(unsigned)stride_grid(slots), kThreads, 0, s>>>(table, slots);
        XRS_CUDA(cudaGetLastError());
        combine_insert<<<(unsigned)grid, kThreads, stage_bytes(K), s>>>(l, K, H, W, table, (uint64_t)slots - 1, flags);
    } else {
        combine_label<<<(unsigned)grid, kThreads, stage_bytes(K), s>>>(
            l, K, H, W, (const long long *)table, (uint64_t)slots - 1, (const long long *)reps, out, out_pitch);
    }
    XRS_CUDA(cudaGetLastError());
    return XRS_OK;
}

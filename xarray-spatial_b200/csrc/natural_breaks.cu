// natural_breaks.cu -- the device work of natural_breaks (classify.py:589-834 of the reference, NumPy path;
// DESIGN.md section 4.11): the reference's seeded sample of cell indices and its Jenks matrices.
//
// The sample.  The reference shuffles np.linspace(0, n, n, dtype=uint32) -- the identity -- with
// RandomState(seed).shuffle and keeps the first s entries.  Only the set matters, and steps i < s only permute
// positions inside [0, s), so it follows from the draws j_i of the steps i >= max(s, 1): first[c] is the smallest
// such step with j_i = c < i, and position q < s ends up holding the index reached by following first[] from q.
// The word stream is generated in chunks of kChunk words, chunk c from the state c kChunk words ahead (jump-ahead,
// mt19937.cuh, by a doubling tree of jumps).  Which step a chunk's first word meets depends on every earlier
// chunk's acceptances, so each chunk counts its acceptances from a guessed first step, a scan turns the counts
// into first steps, and the chunks whose first step changed count again until none does.  Chunk c is exact after
// at most c + 1 rounds; in practice an acceptance count hardly depends on a small error in its first step.
//
// The Jenks matrices.  Cell (l, j) reads only column j - 1 of rows below l and writes only row l, so the columns
// are filled one launch each, every row independent, each running its m-loop in the reference's order with its
// float32 / float64 arithmetic (the build passes -fmad=false; products, sums and the divide are unfused IEEE).
#include <math.h>

#include <algorithm>
#include <mutex>
#include <vector>

#include "common.cuh"
#include "mt19937.cuh"

namespace xrs {
namespace {

using namespace mt;

constexpr int kGenThreads = 640;                  // one per state word, rounded up to whole warps
constexpr int kResolveUnroll = 16;                // words per lane in flight in the resolve
constexpr int kResolveWarps = 4;                  // chunks per resolve CTA
constexpr int64_t kChunkBlocks = 832;             // 624-word blocks per chunk
constexpr int64_t kChunk = kChunkBlocks * kMtN;   // 519168 words, a multiple of 32 * kResolveUnroll
constexpr int kScanThreads = 1024;
constexpr int kCompactThreads = 256, kCompactWords = 16;   // bitmap words per thread of the compaction
constexpr int64_t kCompactTile = (int64_t)kCompactThreads * kCompactWords;
static_assert(kChunk % (32 * kResolveUnroll) == 0, "the resolve reads whole groups of words");

int64_t align256(int64_t b) { return (b + 255) & ~(int64_t)255; }

// The jump polynomials x^(kChunk 2^L) mod phi, L = 0 .. 15, computed once per process.
constexpr int kMaxLevels = 16;
std::once_flag g_poly_once;
std::vector<uint64_t> g_polys;   // kMaxLevels x kPolyWords
int g_poly_deg[kMaxLevels];
bool g_poly_ok = false;

void build_polys() {
    const Poly phi = mt_char_poly();
    if (phi.empty()) return;
    Poly p = poly_x_pow_mod((uint64_t)kChunk, phi);
    g_polys.assign((size_t)kMaxLevels * kPolyWords, 0);
    for (int L = 0; L < kMaxLevels; ++L) {
        std::copy(p.begin(), p.end(), g_polys.begin() + (size_t)L * kPolyWords);
        g_poly_deg[L] = poly_degree(p);
        p = poly_square_mod(p, phi);
    }
    g_poly_ok = true;
}

// Expected words the draws of steps lo .. hi take: step i takes (mask(i) + 1) / (i + 1) on average.
double harmonic(double m) {   // H(m) = sum_{k=1..m} 1 / k
    if (m < 1) return 0.0;
    if (m < 64) {
        double h = 0;
        for (int k = 1; k <= (int)m; ++k) h += 1.0 / k;
        return h;
    }
    return log(m) + 0.57721566490153286 + 1.0 / (2 * m) - 1.0 / (12 * m * m);
}

double expected_words(int64_t lo, int64_t hi) {
    double e = 0;
    for (int b = 0; b < 33 && lo <= hi; ++b) {
        // steps [2^b, 2^(b + 1)) share the mask 2^(b + 1) - 1
        const int64_t a = std::max<int64_t>(lo, (int64_t)1 << b), z = std::min<int64_t>(hi, ((int64_t)2 << b) - 1);
        if (a > z) continue;
        e += (double)((int64_t)2 << b) * (harmonic((double)z + 1) - harmonic((double)a));
    }
    return e;
}

struct SampleLayout {
    int64_t chunks, levels, ctl, polys, states, words, starts, counts, dirty, first, bitmap, blocks, total;
    SampleLayout(int64_t n, int64_t s) {
        const int64_t lo = std::max<int64_t>(s, 1);
        const double steps = (double)(n - lo);
        const double need = expected_words(lo, n - 1) + 8.0 * sqrt(2.0 * steps + 1.0) + 4096.0;
        chunks = std::max<int64_t>(1, (int64_t)ceil(need / (double)kChunk));
        levels = 0;
        while (((int64_t)1 << levels) < chunks) ++levels;
        const int64_t nw = (n + 31) / 32;
        ctl = 0;
        polys = 256;
        states = polys + align256(std::max<int64_t>(levels, 1) * kPolyWords * 8);
        words = states + align256(chunks * kMtN * 4);
        starts = words + align256(chunks * kChunk * 4);
        counts = starts + align256((chunks + 1) * 8);
        dirty = counts + align256(chunks * 8);
        first = dirty + align256(chunks);
        bitmap = first + align256(n * 4);
        blocks = bitmap + align256(nw * 4);
        total = blocks + align256(((nw + kCompactTile - 1) / kCompactTile + 1) * 8);
    }
};

struct SampleCtl {
    int changed;
    int pad;
    int64_t end;   // the step after the last chunk's draws (lo - 1 once the stream reached step lo)
};

__global__ void nb_seed_kernel(uint32_t *state, uint32_t seed) { mt_init(state, seed); }

// states[c] = p(T) states[c - half] for c in [half, min(2 half, C)): Horner over p's coefficients, one warp per
// chunk.  The accumulator is kept relative to its oldest word `idx`; the results sit at a block boundary.
__global__ void __launch_bounds__(32) nb_jump_kernel(uint32_t *states, const uint64_t *poly, int deg, int64_t half,
                                                     int64_t C) {
    const int64_t c = half + blockIdx.x;
    if (c >= C) return;
    __shared__ uint32_t acc[kMtN], src[kMtN];
    const int lane = threadIdx.x;
    for (int j = lane; j < kMtN; j += 32) {
        src[j] = states[(c - half) * kMtN + j];
        acc[j] = 0;
    }
    __syncwarp();
    int idx = 0;
    uint64_t word = poly[deg >> 6];
    for (int k = deg; k >= 0; --k) {
        if ((k & 63) == 63) word = poly[k >> 6];
        if (lane == 0) acc[idx] = mt_twist_word(acc, idx);
        idx = idx + 1 == kMtN ? 0 : idx + 1;
        __syncwarp();
        if ((word >> (k & 63)) & 1u) {
            for (int j = lane; j < kMtN; j += 32) {
                const int e = idx + j;
                acc[e >= kMtN ? e - kMtN : e] ^= src[j];
            }
            __syncwarp();
        }
    }
    for (int j = lane; j < kMtN; j += 32) {
        const int e = idx + j;
        states[c * kMtN + j] = acc[e >= kMtN ? e - kMtN : e];
    }
}

// Chunk c's kChunk tempered words, one CTA per chunk, from its block-boundary state.
__global__ void __launch_bounds__(kGenThreads) nb_gen_kernel(const uint32_t *states, uint32_t *words) {
    __shared__ uint32_t mt[kMtN];
    const int64_t c = blockIdx.x;
    const int t = threadIdx.x;
    if (t < kMtN) mt[t] = states[c * kMtN + t];
    __syncthreads();
    uint32_t *out = words + c * kChunk;
    for (int64_t b = 0; b < kChunkBlocks; ++b) {
        for (int p = 0; p < 4; ++p) {
            const bool mine = t >= phase_begin(p) && t < phase_begin(p + 1);
            const uint32_t nv = mine ? mt_twist_word(mt, t) : 0;
            __syncthreads();   // every read of the phase before any write
            if (mine) mt[t] = nv;
            __syncthreads();
        }
        if (t < kMtN) out[b * kMtN + t] = mt_temper(mt[t]);
    }
}

// The draws of chunk c from its first step starts[c], one warp per chunk, down to step lo: 32 words at a time by
// chunk_uniform / sure_accept with two ballots, word by word at a change of mask, near the end or around an
// undecided word.  COUNT: counts[c] = the steps drawn (dirty chunks only).  Otherwise each drawn step i with j_i < i
// writes first[j_i] = max(first[j_i], n - i): the smallest such step, with 0 for none (n - i >= 1 even at n = 2^32).
template <bool COUNT>
__global__ void __launch_bounds__(32 * kResolveWarps) nb_resolve_kernel(const uint32_t *words, const int64_t *starts,
                                                                        const uint8_t *dirty, int64_t *counts,
                                                                        int64_t C, uint32_t lo, int64_t n,
                                                                        uint32_t *first) {
    const int64_t c = (int64_t)blockIdx.x * kResolveWarps + (threadIdx.x >> 5);
    if (c >= C || (COUNT && !dirty[c])) return;
    const int lane = threadIdx.x & 31;
    const unsigned full = 0xffffffffu, below = (1u << lane) - 1u;
    const int64_t st = starts[c];
    uint32_t i = st < (int64_t)lo ? 0u : (uint32_t)st;
    const bool live = st >= (int64_t)lo;
    const uint32_t *w = words + c * kChunk;
    for (int64_t q = 0; live && i >= lo && q < kChunk; q += 32 * kResolveUnroll) {
        uint32_t r[kResolveUnroll];
#pragma unroll
        for (int u = 0; u < kResolveUnroll; ++u) r[u] = __ldcs(w + q + 32 * u + lane);
#pragma unroll
        for (int u = 0; u < kResolveUnroll; ++u) {
            if (i < lo) break;
            const uint32_t v = r[u] & interval_mask(i);
            const bool fast = chunk_uniform(i) && !__any_sync(full, undecided(v, i));
            if (fast) {
                const bool acc = sure_accept(v, i);
                const unsigned a = __ballot_sync(full, acc);
                if (!COUNT && acc) {
                    const uint32_t step = i - __popc(a & below);
                    if (step >= lo && v != step) atomicMax(first + v, (uint32_t)(n - step));
                }
                i -= __popc(a);   // i >= 32 here, so no wrap; steps below lo are not kept
            } else {
                for (int l = 0; l < 32 && i >= lo; ++l) {
                    const uint32_t vl = __shfl_sync(full, r[u], l) & interval_mask(i);
                    if (vl <= i) {
                        if (!COUNT && lane == 0 && vl != i) atomicMax(first + vl, (uint32_t)(n - i));
                        --i;
                    }
                }
            }
        }
    }
    if (COUNT && lane == 0) counts[c] = live ? st - max((int64_t)i, (int64_t)lo - 1) : 0;
}

// Block-wide exclusive scan of one int64 per thread; returns the block total through *total.
__device__ int64_t block_exclusive_scan(int64_t v, int64_t *total) {
    __shared__ int64_t warp_sums[32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    int64_t x = v;
    for (int d = 1; d < 32; d <<= 1) {
        const int64_t y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= d) x += y;
    }
    if (lane == 31) warp_sums[wid] = x;
    __syncthreads();
    if (wid == 0) {
        int64_t s = lane < nwarps ? warp_sums[lane] : 0;
        for (int d = 1; d < 32; d <<= 1) {
            const int64_t y = __shfl_up_sync(0xffffffffu, s, d);
            if (lane >= d) s += y;
        }
        if (lane < nwarps) warp_sums[lane] = s;   // inclusive
    }
    __syncthreads();
    const int64_t before = (wid ? warp_sums[wid - 1] : 0) + x - v;
    *total = warp_sums[nwarps - 1];
    __syncthreads();
    return before;
}

// starts[c] = max(n - 1 - sum of counts before c, lo - 1); dirty[c] marks the chunks whose first step moved.
__global__ void __launch_bounds__(kScanThreads) nb_starts_kernel(int64_t *starts, const int64_t *counts,
                                                                 uint8_t *dirty, int64_t C, int64_t n, int64_t lo,
                                                                 SampleCtl *ctl) {
    int64_t carry = 0;
    int changed = 0;
    for (int64_t base = 0; base < C; base += kScanThreads) {
        const int64_t c = base + threadIdx.x;
        int64_t total;
        const int64_t before = block_exclusive_scan(c < C ? counts[c] : 0, &total);
        if (c < C) {
            const int64_t s = max(n - 1 - (carry + before), lo - 1);
            const bool moved = s != starts[c];
            dirty[c] = moved;
            changed |= moved;
            starts[c] = s;
        }
        carry += total;
    }
    changed = __syncthreads_or(changed);
    if (threadIdx.x == 0) {
        ctl->changed = changed;
        ctl->end = max(n - 1 - carry, lo - 1);
    }
}

// Position q < s ends up holding the index reached by following first[] from q; mark it in the bitmap.
__global__ void nb_chains_kernel(const uint32_t *first, int64_t n, int64_t s, uint32_t *bitmap) {
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < s; q += (int64_t)gridDim.x * blockDim.x) {
        int64_t x = q;
        for (uint32_t e = first[x]; e != 0; e = first[x]) x = n - (int64_t)e;
        atomicOr(bitmap + (x >> 5), 1u << (x & 31));
    }
}

__global__ void __launch_bounds__(kCompactThreads) nb_bitcount_kernel(const uint32_t *bitmap, int64_t nw,
                                                                      int64_t *blocks) {
    const int64_t w0 = (int64_t)blockIdx.x * kCompactTile + (int64_t)threadIdx.x * kCompactWords;
    int64_t cnt = 0;
    for (int k = 0; k < kCompactWords; ++k)
        if (w0 + k < nw) cnt += __popc(bitmap[w0 + k]);
    int64_t total;
    block_exclusive_scan(cnt, &total);
    if (threadIdx.x == 0) blocks[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kScanThreads) nb_block_scan_kernel(int64_t *blocks, int64_t nb) {
    int64_t carry = 0;
    for (int64_t base = 0; base < nb; base += kScanThreads) {
        const int64_t b = base + threadIdx.x;
        int64_t total;
        const int64_t before = block_exclusive_scan(b < nb ? blocks[b] : 0, &total);
        if (b < nb) blocks[b] = carry + before;
        carry += total;
    }
}

// The marked indices in ascending order.
__global__ void __launch_bounds__(kCompactThreads) nb_compact_kernel(const uint32_t *bitmap, int64_t nw,
                                                                     const int64_t *blocks, int64_t *out) {
    const int64_t w0 = (int64_t)blockIdx.x * kCompactTile + (int64_t)threadIdx.x * kCompactWords;
    int64_t cnt = 0;
    for (int k = 0; k < kCompactWords; ++k)
        if (w0 + k < nw) cnt += __popc(bitmap[w0 + k]);
    int64_t total;
    int64_t pos = blocks[blockIdx.x] + block_exclusive_scan(cnt, &total);
    for (int k = 0; k < kCompactWords; ++k) {
        if (w0 + k >= nw) break;
        for (uint32_t b = bitmap[w0 + k]; b; b &= b - 1) out[pos++] = (w0 + k) * 32 + __ffs(b) - 1;
    }
}

int64_t stride_grid(int64_t n) {
    return std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, (int64_t)sm_count() * 8));
}

int sample_args(int64_t n, int64_t s) {
    XRS_REQUIRE(n >= 1, "the sample needs at least one cell");
    if (n > ((int64_t)1 << 32)) {
        set_error("natural_breaks samples rasters of at most 2^32 cells (this one has %lld): beyond that the "
                  "reference's uint32 index array wraps", (long long)n);
        return XRS_EINVAL;
    }
    XRS_REQUIRE(s >= 1 && s < n, "the sample size must be 1 .. n - 1");
    return XRS_OK;
}

// ---------------------------------------------------------------------------------------------- Jenks
// Row l of column j (2 .. k; j = 1: the full-prefix variance).  x: the sorted sample as float32.
template <bool FIRST>
__device__ __forceinline__ void jenks_row(const float *__restrict__ x, int64_t l, int64_t n, int j,
                                          float *__restrict__ lcl, float *__restrict__ var) {
    const int64_t ld = n + 1;
    const float *prev = var + (int64_t)(j - 1) * ld;
    double sum = 0.0, sum_squares = 0.0, w = 0.0, variance = 0.0;
    float best = INFINITY, limit = 0.0f;
    for (int64_t m = 0; m < l; ++m) {
        const int64_t i4 = l - m - 1;
        const float val = x[i4];
        w = __dadd_rn(w, 1.0);
        sum = __dadd_rn(sum, (double)val);
        sum_squares = __dadd_rn(sum_squares, (double)__fmul_rn(val, val));
        variance = __dsub_rn(sum_squares, __ddiv_rn(__dmul_rn(sum, sum), w));
        if (FIRST || i4 == 0) continue;
        const double nv = __dadd_rn(variance, (double)prev[i4]);
        if ((double)best >= nv) {
            limit = (float)(l - m);
            best = __double2float_rn(nv);
        }
    }
    if (FIRST) {
        lcl[ld + l] = 1.0f;
        var[ld + l] = __double2float_rn(variance);
    } else {
        lcl[(int64_t)j * ld + l] = limit;
        var[(int64_t)j * ld + l] = best;
    }
}

// Rows 2 .. n, thread t taking rows 2 + t and n - t, so every thread runs n + 2 iterations.
template <bool FIRST>
__global__ void __launch_bounds__(128) nb_jenks_column_kernel(const float *__restrict__ x, int64_t n, int j,
                                                              float *__restrict__ lcl, float *__restrict__ var) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t a = 2 + t, b = n - t;
    if (a > b) return;
    jenks_row<FIRST>(x, a, n, j, lcl, var);
    if (b != a) jenks_row<FIRST>(x, b, n, j, lcl, var);
}

// The matrices' initial values: lcl row 1 = 1 in columns >= 1, var rows >= 2 = inf in columns >= 1, else 0.
__global__ void nb_jenks_init_kernel(int64_t n, int k, float *lcl, float *var) {
    const int64_t ld = n + 1, total = (int64_t)(k + 1) * ld;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t j = e / ld, l = e - j * ld;
        lcl[e] = (l == 1 && j >= 1) ? 1.0f : 0.0f;
        var[e] = (l >= 2 && j >= 1) ? INFINITY : 0.0f;
    }
}

}  // namespace
}  // namespace xrs

using namespace xrs;

extern "C" int xrs_nb_sample_scratch_bytes(int64_t n, int64_t s, int64_t *bytes) {
    XRS_REQUIRE(bytes != nullptr, "NULL pointer");
    const int rc = sample_args(n, s);
    if (rc) return rc;
    *bytes = SampleLayout(n, s).total;
    return XRS_OK;
}

extern "C" int xrs_nb_sample(int64_t n, int64_t s, uint32_t seed, int64_t *out, void *scratch, int64_t scratch_bytes,
                             int64_t *rounds, xrs_stream_t stream) {
    int rc = sample_args(n, s);
    if (rc) return rc;
    XRS_REQUIRE(out != nullptr, "NULL output");
    XRS_REQUIRE(scratch != nullptr, "NULL scratch buffer");
    const SampleLayout L(n, s);
    if (scratch_bytes < L.total) {
        set_error("scratch buffer of %lld bytes is too small: this call needs %lld (xrs_nb_sample_scratch_bytes)",
                  (long long)scratch_bytes, (long long)L.total);
        return XRS_EINVAL;
    }
    if (L.levels > kMaxLevels) {
        set_error("xrs_nb_sample: %lld chunks need more than %d jump levels", (long long)L.chunks, kMaxLevels);
        return XRS_EINVAL;
    }
    std::call_once(g_poly_once, build_polys);
    if (!g_poly_ok) {
        set_error("xrs_nb_sample: Berlekamp-Massey did not find MT19937's degree-19937 polynomial (internal error)");
        return XRS_ECUDA;
    }
    cudaStream_t st = (cudaStream_t)stream;
    char *sc = (char *)scratch;
    SampleCtl *ctl = (SampleCtl *)(sc + L.ctl);
    uint64_t *polys = (uint64_t *)(sc + L.polys);
    uint32_t *states = (uint32_t *)(sc + L.states), *words = (uint32_t *)(sc + L.words);
    int64_t *starts = (int64_t *)(sc + L.starts), *counts = (int64_t *)(sc + L.counts);
    uint8_t *dirty = (uint8_t *)(sc + L.dirty);
    uint32_t *first = (uint32_t *)(sc + L.first), *bitmap = (uint32_t *)(sc + L.bitmap);
    int64_t *blocks = (int64_t *)(sc + L.blocks);
    const int64_t C = L.chunks, lo = std::max<int64_t>(s, 1);

    // the jump and the generation
    if (L.levels)
        XRS_CUDA(cudaMemcpyAsync(polys, g_polys.data(), (size_t)L.levels * kPolyWords * 8, cudaMemcpyHostToDevice, st));
    nb_seed_kernel<<<1, 1, 0, st>>>(states, seed);
    XRS_CUDA(cudaGetLastError());
    for (int lev = 0; lev < L.levels; ++lev) {
        const int64_t half = (int64_t)1 << lev;
        nb_jump_kernel<<<(unsigned)std::min(half, C - half), 32, 0, st>>>(states, polys + (int64_t)lev * kPolyWords,
                                                                         g_poly_deg[lev], half, C);
        XRS_CUDA(cudaGetLastError());
    }
    nb_gen_kernel<<<(unsigned)C, kGenThreads, 0, st>>>(states, words);
    XRS_CUDA(cudaGetLastError());

    // the resolve: first steps guessed from the expected words per step, then counted and re-scanned until fixed
    std::vector<int64_t> guess(C + 1);
    {
        int64_t hi = n - 1;
        for (int64_t c = 0; c < C; ++c) {
            guess[c] = hi;
            // the step at which the expected words from hi on reach kChunk (bisection on the expectation)
            int64_t a = lo - 1, b = hi;
            while (a < b) {
                const int64_t mid = a + (b - a + 1) / 2;
                if (expected_words(mid, hi) >= (double)kChunk) a = mid;
                else b = mid - 1;
            }
            hi = std::max<int64_t>(a, lo - 1);
        }
    }
    XRS_CUDA(cudaMemcpyAsync(starts, guess.data(), C * 8, cudaMemcpyHostToDevice, st));
    XRS_CUDA(cudaMemsetAsync(dirty, 1, C, st));
    const unsigned rgrid = (unsigned)((C + kResolveWarps - 1) / kResolveWarps);
    int64_t round = 0;
    SampleCtl h{};
    for (;;) {
        nb_resolve_kernel<true><<<rgrid, 32 * kResolveWarps, 0, st>>>(words, starts, dirty, counts, C, (uint32_t)lo,
                                                                      n, nullptr);
        XRS_CUDA(cudaGetLastError());
        nb_starts_kernel<<<1, kScanThreads, 0, st>>>(starts, counts, dirty, C, n, lo, ctl);
        XRS_CUDA(cudaGetLastError());
        XRS_CUDA(cudaMemcpyAsync(&h, ctl, sizeof(h), cudaMemcpyDeviceToHost, st));
        XRS_CUDA(cudaStreamSynchronize(st));
        ++round;
        if (!h.changed) break;
        if (round > C + 1) {
            set_error("xrs_nb_sample: the chunk starts did not settle in %lld rounds (internal error)", (long long)round);
            return XRS_ECUDA;
        }
    }
    if (h.end != lo - 1) {
        set_error("xrs_nb_sample: %lld words did not reach step %lld (internal error)", (long long)(C * kChunk),
                  (long long)lo);
        return XRS_ECUDA;
    }

    // first[], the chains and the sorted set
    XRS_CUDA(cudaMemsetAsync(first, 0, n * 4, st));
    nb_resolve_kernel<false><<<rgrid, 32 * kResolveWarps, 0, st>>>(words, starts, dirty, counts, C, (uint32_t)lo, n,
                                                                   first);
    XRS_CUDA(cudaGetLastError());
    const int64_t nw = (n + 31) / 32, nb = (nw + kCompactTile - 1) / kCompactTile;
    XRS_CUDA(cudaMemsetAsync(bitmap, 0, nw * 4, st));
    nb_chains_kernel<<<(unsigned)stride_grid(s), 256, 0, st>>>(first, n, s, bitmap);
    XRS_CUDA(cudaGetLastError());
    nb_bitcount_kernel<<<(unsigned)nb, kCompactThreads, 0, st>>>(bitmap, nw, blocks);
    XRS_CUDA(cudaGetLastError());
    nb_block_scan_kernel<<<1, kScanThreads, 0, st>>>(blocks, nb);
    XRS_CUDA(cudaGetLastError());
    nb_compact_kernel<<<(unsigned)nb, kCompactThreads, 0, st>>>(bitmap, nw, blocks, out);
    XRS_CUDA(cudaGetLastError());
    if (rounds) *rounds = round;
    return XRS_OK;
}

extern "C" int xrs_nb_jenks_scratch_bytes(int64_t n, int k, int64_t *bytes) {
    XRS_REQUIRE(bytes != nullptr, "NULL pointer");
    XRS_REQUIRE(n >= 1 && k >= 1, "the Jenks matrices need n >= 1 values and k >= 1 classes");
    *bytes = align256((int64_t)(k + 1) * (n + 1) * 4);
    return XRS_OK;
}

extern "C" int xrs_nb_jenks(const float *x, int64_t n, int k, float *lcl, void *scratch, int64_t scratch_bytes,
                            xrs_stream_t stream) {
    XRS_REQUIRE(n >= 1 && k >= 1, "the Jenks matrices need n >= 1 values and k >= 1 classes");
    XRS_REQUIRE(x != nullptr && lcl != nullptr && scratch != nullptr, "NULL pointer");
    int64_t need = 0;
    xrs_nb_jenks_scratch_bytes(n, k, &need);
    if (scratch_bytes < need) {
        set_error("scratch buffer of %lld bytes is too small: this call needs %lld (xrs_nb_jenks_scratch_bytes)",
                  (long long)scratch_bytes, (long long)need);
        return XRS_EINVAL;
    }
    cudaStream_t st = (cudaStream_t)stream;
    float *var = (float *)scratch;
    nb_jenks_init_kernel<<<(unsigned)stride_grid((int64_t)(k + 1) * (n + 1)), 256, 0, st>>>(n, k, lcl, var);
    XRS_CUDA(cudaGetLastError());
    const int64_t rows = n - 1, threads = (rows + 1) / 2;
    if (threads <= 0) return XRS_OK;
    const unsigned grid = (unsigned)((threads + 127) / 128);
    nb_jenks_column_kernel<true><<<grid, 128, 0, st>>>(x, n, 1, lcl, var);
    XRS_CUDA(cudaGetLastError());
    for (int j = 2; j <= k; ++j) {
        nb_jenks_column_kernel<false><<<grid, 128, 0, st>>>(x, n, j, lcl, var);
        XRS_CUDA(cudaGetLastError());
    }
    return XRS_OK;
}

// H100 ceiling probe and geometry sweep of stencil3_tma_kernel (csrc/stencil3.cuh), 32768^2 float32.
//
//  (1) the copy ceiling of this card: cudaMemcpy device-to-device, a float4 grid-stride copy kernel, and a
//      no-op copy operator (CopyOp) pushed through the 3x3 skeleton with either epilogue -- the per-warp
//      register stores (st.global.cs.v4) and the bulk-store epilogue (staging in shared memory, one
//      cp.async.bulk per tile row issued by a store warp);
//  (2) the flagship operators (square-cell slope, hillshade, focal.mean f32) over ROWS x STAGES x WARPS x
//      CTAs per SM with both epilogues, then the other float32 operators of surface.cu's geometry();
//  (1c) where the input boxes start: the shipped 32-byte halo (every box row starts on an L2 sector) against
//      a 16-byte halo (every float32 box row starts 16 B into a sector), alternating, for the no-op operator and
//      the flagship three and the 4-output suite; as the control, a float64 copy with its 32-byte halo read from an aligned base and
//      from a base 16 B further on;
//  (3) outputs of the two epilogues, and of the two halo widths, compared bit for bit at the shipped geometries.
// Every line: CUDA-event median of 9 launches (after 2 warm-ups), GB/s of algorithmic bytes, fraction of
// the 3.35 TB/s data sheet and of the best copy measured in (1).  nvidia-smi is sampled every 50 ms in the
// background; each section prints the median SM clock and how many samples showed an active power cap.
//
// `tune5 align` runs (1), (1c) with 6 rounds instead of 3, and (3).
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -fmad=false -DXRS_BUILD \
//        -o tune5 scripts/tune/tune5.cu xarray-spatial_b200/csrc/lib_core.cu
#include <signal.h>
#include <sys/prctl.h>
#include <sys/wait.h>
#include <unistd.h>

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../xarray-spatial_b200/csrc/surface_ops.cuh"
using namespace xrs;

static const double kDataSheetGBs = 3350.0;
static double g_best_copy = 0.0;  // GB/s, set by section (1)

// ------------------------------------------------------------------ nvidia-smi sampler (child process)
struct SmiSampler {
    pid_t pid = -1;
    int fd = -1;
    std::thread reader;
    std::mutex mu;
    std::vector<std::string> rows;
    void start() {
        int p[2];
        if (pipe(p) != 0) return;
        pid = fork();
        if (pid == 0) {
            prctl(PR_SET_PDEATHSIG, SIGTERM);  // never outlive the probe
            dup2(p[1], 1);
            close(p[0]);
            execlp("nvidia-smi", "nvidia-smi",
                   "--query-gpu=clocks.sm,power.draw,clocks_event_reasons.sw_power_cap,"
                   "clocks_event_reasons.hw_slowdown,clocks_event_reasons.sw_thermal_slowdown",
                   "--format=csv,noheader,nounits", "-lms", "50", (char *)nullptr);
            _exit(127);
        }
        close(p[1]);
        fd = p[0];
        reader = std::thread([this] {
            FILE *f = fdopen(fd, "r");
            char line[512];
            while (f && fgets(line, sizeof line, f)) {
                std::lock_guard<std::mutex> g(mu);
                rows.emplace_back(line);
            }
            if (f) fclose(f);
        });
    }
    size_t mark() {
        std::lock_guard<std::mutex> g(mu);
        return rows.size();
    }
    // median SM clock, samples with sw_power_cap / any slowdown active, in rows [a, b)
    void summary(const char *what, size_t a, size_t b) {
        std::vector<double> mhz, watts;
        int cap = 0, slow = 0, n = 0;
        {
            std::lock_guard<std::mutex> g(mu);
            for (size_t i = a; i < b && i < rows.size(); ++i) {
                char c1[64] = "", c2[64] = "", c3[64] = "";
                double m = 0, w = 0;
                if (sscanf(rows[i].c_str(), "%lf, %lf, %63[^,], %63[^,], %63s", &m, &w, c1, c2, c3) < 5) continue;
                ++n;
                mhz.push_back(m);
                watts.push_back(w);
                if (strncmp(c1, "Active", 6) == 0) ++cap;
                if (strncmp(c2, "Active", 6) == 0 || strncmp(c3, "Active", 6) == 0) ++slow;
            }
        }
        if (!n) { printf("# clocks [%s]: no nvidia-smi samples\n", what); return; }
        std::sort(mhz.begin(), mhz.end());
        std::sort(watts.begin(), watts.end());
        printf("# clocks [%s]: %d samples, SM clock median %.0f MHz (min %.0f), power median %.0f W (max %.0f), "
               "sw_power_cap active in %d, hw/thermal slowdown in %d\n",
               what, n, mhz[n / 2], mhz[0], watts[n / 2], watts[n - 1], cap, slow);
        fflush(stdout);
    }
    void stop() {
        if (pid > 0) {
            kill(pid, SIGTERM);
            waitpid(pid, nullptr, 0);
        }
        if (reader.joinable()) reader.join();
    }
};

static void print_card() {
    FILE *f = popen("nvidia-smi --query-gpu=name,power.limit,clocks.max.sm,clocks.sm,memory.total,driver_version "
                    "--format=csv", "r");
    char line[512];
    while (f && fgets(line, sizeof line, f)) printf("# %s", line);
    if (f) pclose(f);
    fflush(stdout);
}

// ------------------------------------------------------------------ workloads
__global__ void fill(float *p, size_t n, int W) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    for (; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float x = (float)(i % W), y = (float)(i / W);
        p[i] = 2000.f + 900.f * __sinf(x * 0.0013f) * __cosf(y * 0.0011f) + 35.f * __sinf(x * 0.071f + y * 0.053f);
    }
}
__global__ void widen(const float *a, double *b, size_t n) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    for (; i < n; i += (size_t)gridDim.x * blockDim.x) b[i] = (double)a[i];
}
__global__ void copyk(const float4 *a, float4 *b, size_t n4) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    for (; i < n4; i += (size_t)gridDim.x * blockDim.x) b[i] = a[i];
}
__global__ void count_diff(const unsigned *a, const unsigned *b, size_t n, unsigned long long *cnt) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    unsigned long long c = 0;
    for (; i < n; i += (size_t)gridDim.x * blockDim.x) c += a[i] != b[i];
    if (c) atomicAdd(cnt, c);
}

// The skeleton with nothing to compute: output row y-1 = input row y-1.
template <typename T> struct CopyOpT {
    using in_t = T;
    using out_t = T;
    static constexpr int kOutputs = 1;
    struct Params { int unused; };
    T r1[4];
    __device__ explicit CopyOpT(const Params &) { r1[0] = r1[1] = r1[2] = r1[3] = T(0); }
    __device__ __forceinline__ void step(const Row6<T> &row, Vec4<T> (&out)[1]) {
#pragma unroll
        for (int i = 0; i < 4; ++i) { out[0].v[i] = r1[i]; r1[i] = row.c[i]; }
    }
};
using CopyOp = CopyOpT<float>;
using CopyOpD = CopyOpT<double>;

static cudaEvent_t e0, e1;
template <typename F> float time_it(F f, int reps = 9) {
    for (int i = 0; i < 2; ++i) f();
    std::vector<float> t;
    for (int i = 0; i < reps; ++i) {
        cudaEventRecord(e0); f(); cudaEventRecord(e1); cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1); t.push_back(ms);
    }
    if (cudaGetLastError() != cudaSuccess) return -2.f;
    std::sort(t.begin(), t.end());
    return t[t.size() / 2];
}

// n/a codes: -1 does not fit (shared memory / occupancy below CTAS), -2 CUDA error, -3 no tensor map.
// PAD = halo cells; `shift` > 0 reads the raster from `shift` cells past its base (W - 4 cells wide).
template <typename Op, int ROWS, int STAGES, int WARPS, int CTAS, bool BULK, int PAD = SrcPad<typename Op::in_t>::value>
float run(const typename Op::in_t *in, typename Op::out_t *const *outp, int64_t H, int64_t W,
          const typename Op::Params &prm, int shift = 0) {
    using T = typename Op::in_t;
    using Cfg = TmaCfg<Op, ROWS, STAGES, WARPS, CTAS, T, PAD>;
    if constexpr (BULK && !Cfg::kBulk) {
        return -1.f;
    } else {
        CUtensorMap tmap;
        const int64_t pitch = W * sizeof(T);
        if (shift) W -= 4;
        if (!make_tensor_map_2d(&tmap, in + shift, pitch, H, W, dtype_of<T>(), kSubW, ROWS)) return -3.f;
        OutPtrs<Op> outs;
        for (int k = 0; k < Op::kOutputs; ++k) outs.p[k] = outp[k];
        outs.pitch_elems = pitch / sizeof(T);
        constexpr size_t smem = BULK ? Cfg::kBulkSmem : Cfg::kRegSmem;
        constexpr int threads = (WARPS + 1 + (BULK ? 1 : 0)) * 32;
        auto kern = stencil3_tma_kernel<Op, ROWS, STAGES, WARPS, T, PAD, BULK>;
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
            cudaGetLastError();
            return -1.f;
        }
        int occ = 0;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, threads, smem);
        if (occ < CTAS) return -1.f;
        return time_it([&] { launch_tma<Op, ROWS, STAGES, WARPS, CTAS, T, PAD, BULK>(tmap, prm, outs, H, W, 0, kStripTma); });
    }
}

static void report(const char *name, const char *cfg, float ms, double bytes) {
    if (ms < 0) { printf("%-16s %-30s : n/a (%d)\n", name, cfg, (int)ms); fflush(stdout); return; }
    const double gbs = bytes / (ms * 1e-3) / 1e9;
    printf("%-16s %-30s : %7.3f ms %6.0f GB/s  %.3f of 3.35 TB/s  %.3f of best copy\n", name, cfg, ms, gbs,
           gbs / kDataSheetGBs, g_best_copy > 0 ? gbs / g_best_copy : 0.0);
    fflush(stdout);
}

int main(int argc, char **argv) {
    const bool align_only = argc > 1 && strcmp(argv[1], "align") == 0;  // sections (1), (1c) and (3) only
    const int64_t H = 32768, W = 32768;
    const size_t n = (size_t)H * W;
    print_card();
    SmiSampler smi;
    smi.start();
    float *in, *o[4], *oref;
    double *ind, *od;
    cudaMalloc(&in, n * 4);
    for (int k = 0; k < 4; ++k) cudaMalloc(&o[k], n * 4);
    cudaMalloc(&oref, n * 4);
    cudaMalloc(&ind, n * 4);  // f64 rasters: half the rows
    cudaMalloc(&od, n * 8);
    fill<<<132 * 8, 256>>>(in, n, (int)W);
    widen<<<132 * 8, 256>>>(in, ind, n / 2);
    cudaDeviceSynchronize();
    if (cudaGetLastError() != cudaSuccess) { printf("setup failed\n"); smi.stop(); return 1; }
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    const double B8 = 8.0 * n;
    char cfg[96];

    // ---- (1) copy ceiling
    size_t m0 = smi.mark();
    {
        float best = 1e30f, t;
        t = time_it([&] { cudaMemcpyAsync(o[0], in, n * 4, cudaMemcpyDeviceToDevice); }, 15);
        report("cudaMemcpy", "D2D", t, B8); best = std::min(best, t);
        for (int per_sm : {4, 8, 16, 32}) {
            snprintf(cfg, sizeof cfg, "float4 grid-stride %dx%dx256", sm_count(), per_sm);
            t = time_it([&] { copyk<<<sm_count() * per_sm, 256>>>((const float4 *)in, (float4 *)o[0], n / 4); }, 15);
            report("copy kernel", cfg, t, B8); best = std::min(best, t);
        }
        g_best_copy = B8 / (best * 1e-3) / 1e9;
        printf("# best copy: %.3f ms = %.0f GB/s = %.3f of the 3.35 TB/s data sheet\n", best, g_best_copy,
               g_best_copy / kDataSheetGBs);
    }
    smi.summary("copies", m0, smi.mark());

    HillshadeOp::Params hp = {0.42f, 0.2f, -0.3f};
    SlopeParams sp = {1.0, 1.7e-5f};
    SlopeParams sp2 = {1.25, 1.7e-5f};
    AspectOp::Params ap = {0};
    CurvatureOp::Params cp = {100.0 / 900.0};
    CopyOp::Params np_ = {0};
    CopyOpD::Params npd = {0};
    using FM = FocalMeanOp<float, float, false>;
    using FMD = FocalMeanOp<float, double, false>;
    using FDD = FocalMeanOp<double, double, false>;
    FM::Params fp; memset(&fp, 0, sizeof(fp)); fp.ex_nan = 1;
    FMD::Params fdp; memset(&fdp, 0, sizeof(fdp)); fdp.ex_nan = 1;
    FDD::Params fddp; memset(&fddp, 0, sizeof(fddp)); fddp.ex_nan = 1;
    SuiteParams up; up.slope = sp; up.curv = cp; up.hill = hp;
    Conv3Op::Params c3; for (int i = 0; i < 9; ++i) c3.w[i] = 0.1 * (i + 1);
    float *o1[1] = {o[0]};
    float *oref1[1] = {oref};
    double *od1[1] = {od};
    float *o4[4] = {o[0], o[1], o[2], o[3]};

#define RUN(NAME, OP, IN, OUT, HH, PRM, R, S, WP, P, BULK, BYTES) { \
        snprintf(cfg, sizeof cfg, "%s r%d s%d warps=%d cta/sm=%d", BULK ? "bulk" : "reg ", R, S, WP, P); \
        report(NAME, cfg, run<OP, R, S, WP, P, BULK>(IN, OUT, HH, W, PRM), BYTES); }
#define BOTH(NAME, OP, IN, OUT, HH, PRM, R, S, WP, P, BYTES) \
        RUN(NAME, OP, IN, OUT, HH, PRM, R, S, WP, P, false, BYTES) RUN(NAME, OP, IN, OUT, HH, PRM, R, S, WP, P, true, BYTES)
#define SWEEP(NAME, OP, PRM) { size_t a = smi.mark(); \
        BOTH(NAME, OP, in, o1, H, PRM, 2, 4, 16, 1, B8) BOTH(NAME, OP, in, o1, H, PRM, 4, 3, 8, 2, B8) \
        BOTH(NAME, OP, in, o1, H, PRM, 2, 4, 8, 2, B8) BOTH(NAME, OP, in, o1, H, PRM, 4, 2, 8, 2, B8) \
        BOTH(NAME, OP, in, o1, H, PRM, 4, 4, 8, 2, B8) BOTH(NAME, OP, in, o1, H, PRM, 2, 6, 8, 2, B8) \
        BOTH(NAME, OP, in, o1, H, PRM, 4, 4, 8, 1, B8) BOTH(NAME, OP, in, o1, H, PRM, 2, 8, 8, 1, B8) \
        BOTH(NAME, OP, in, o1, H, PRM, 2, 4, 8, 3, B8) BOTH(NAME, OP, in, o1, H, PRM, 2, 6, 16, 1, B8) \
        BOTH(NAME, OP, in, o1, H, PRM, 4, 3, 16, 1, B8) BOTH(NAME, OP, in, o1, H, PRM, 4, 4, 16, 1, B8) \
        BOTH(NAME, OP, in, o1, H, PRM, 2, 3, 16, 2, B8) BOTH(NAME, OP, in, o1, H, PRM, 4, 3, 12, 1, B8) \
        BOTH(NAME, OP, in, o1, H, PRM, 8, 2, 16, 1, B8) BOTH(NAME, OP, in, o1, H, PRM, 8, 2, 8, 2, B8) \
        smi.summary(NAME, a, smi.mark()); }

    // ---- (1c) box alignment, alternating: 16-byte halo (PAD 4) against the shipped 32-byte halo (PAD 8),
    //      shipped float32 geometry; float64 copy, shipped float64 geometry, from 32 B (sector-aligned) and 16 B past the base
    {
        size_t a = smi.mark();
        const double B16s = 16.0 * (H / 2) * (W - 4);
#define ALIGN(NAME, OP, PRM) \
        report(NAME, "halo 16 B bulk r4 s3 warps=16", run<OP, 4, 3, 16, 1, true, 4>(in, o1, H, W, PRM), B8); \
        report(NAME, "halo 32 B bulk r4 s3 warps=16", run<OP, 4, 3, 16, 1, true, 8>(in, o1, H, W, PRM), B8);
        for (int rep = 0; rep < (align_only ? 6 : 3); ++rep) {
            ALIGN("copyop", CopyOp, np_)
            ALIGN("slope(square)", SlopeSqOp, sp)
            ALIGN("hillshade", HillshadeOp, hp)
            ALIGN("focal.mean f32", FM, fp)
            report("suite4", "halo 16 B reg  r8 s2 warps=12", run<SuiteSqOp, 8, 2, 12, 1, false, 4>(in, o4, H, W, up), 20.0 * n);
            report("suite4", "halo 32 B reg  r8 s2 warps=12", run<SuiteSqOp, 8, 2, 12, 1, false, 8>(in, o4, H, W, up), 20.0 * n);
            report("copyop f64", "base +32 B bulk r2 s4 warps=16", run<CopyOpD, 2, 4, 16, 1, true>(ind, od1, H / 2, W, npd, 4), B16s);
            report("copyop f64", "base +16 B bulk r2 s4 warps=16", run<CopyOpD, 2, 4, 16, 1, true>(ind, od1, H / 2, W, npd, 2), B16s);
        }
        smi.summary("alignment", a, smi.mark());
    }

    // ---- (1b) the skeleton's copy operator, then (2) the flagship operators
    if (!align_only) {
        SWEEP("copyop", CopyOp, np_)
        SWEEP("slope(square)", SlopeSqOp, sp)
        SWEEP("hillshade", HillshadeOp, hp)
        SWEEP("focal.mean f32", FM, fp)

        // ---- (2b) the other float32 operators of surface.cu's geometry()
#define OTHER(NAME, OP, IN, OUT, HH, PRM, BYTES) { size_t a = smi.mark(); \
            BOTH(NAME, OP, IN, OUT, HH, PRM, 2, 4, 16, 1, BYTES) BOTH(NAME, OP, IN, OUT, HH, PRM, 4, 3, 8, 2, BYTES) \
            BOTH(NAME, OP, IN, OUT, HH, PRM, 4, 4, 8, 1, BYTES) BOTH(NAME, OP, IN, OUT, HH, PRM, 4, 3, 16, 1, BYTES) \
            BOTH(NAME, OP, IN, OUT, HH, PRM, 2, 4, 8, 2, BYTES) BOTH(NAME, OP, IN, OUT, HH, PRM, 8, 2, 16, 1, BYTES) \
            BOTH(NAME, OP, IN, OUT, HH, PRM, 4, 2, 8, 2, BYTES) BOTH(NAME, OP, IN, OUT, HH, PRM, 2, 4, 8, 1, BYTES) \
            smi.summary(NAME, a, smi.mark()); }
        OTHER("slope(rxy)", SlopeOp, in, o1, H, sp2, B8)
        OTHER("aspect", AspectOp, in, o1, H, ap, B8)
        OTHER("curvature", CurvatureOp, in, o1, H, cp, B8)
        OTHER("conv3", Conv3Op, in, o1, H, c3, B8)
        OTHER("focal f32->f64", FMD, in, od1, H / 2, fdp, 12.0 * (n / 2))
        OTHER("focal.mean f64", FDD, ind, od1, H / 2, fddp, 16.0 * (n / 2))
        {
            size_t a = smi.mark();
            BOTH("suite4", SuiteSqOp, in, o4, H, up, 8, 2, 12, 1, 20.0 * n)
            BOTH("suite4", SuiteSqOp, in, o4, H, up, 2, 4, 8, 1, 20.0 * n)
            BOTH("suite4", SuiteSqOp, in, o4, H, up, 2, 4, 12, 1, 20.0 * n)
            BOTH("suite4", SuiteSqOp, in, o4, H, up, 4, 3, 8, 1, 20.0 * n)
            BOTH("suite4", SuiteSqOp, in, o4, H, up, 2, 3, 16, 1, 20.0 * n)
            BOTH("suite4", SuiteSqOp, in, o4, H, up, 4, 2, 12, 1, 20.0 * n)
            smi.summary("suite4", a, smi.mark());
        }
    }  // !align_only

    // ---- (3) the two epilogues agree bit for bit (shipped geometries)
    unsigned long long *cnt;
    cudaMalloc(&cnt, 8);
    auto diff = [&](const char *name) {
        cudaMemset(cnt, 0, 8);
        count_diff<<<132 * 8, 256>>>((const unsigned *)o[0], (const unsigned *)oref, n, cnt);
        unsigned long long h = 0;
        cudaMemcpy(&h, cnt, 8, cudaMemcpyDeviceToHost);
        printf("bulk vs register epilogue, %-14s: %llu cells differ (%s)\n", name, h, cudaGetErrorString(cudaGetLastError()));
        fflush(stdout);
    };
    cudaMemset(o[0], 0xff, n * 4); cudaMemset(oref, 0, n * 4);
    run<SlopeSqOp, 4, 3, 8, 2, false>(in, oref1, H, W, sp); run<SlopeSqOp, 4, 3, 8, 2, true>(in, o1, H, W, sp); diff("slope(square)");
    run<HillshadeOp, 2, 4, 16, 1, false>(in, oref1, H, W, hp); run<HillshadeOp, 2, 4, 16, 1, true>(in, o1, H, W, hp); diff("hillshade");
    run<FM, 2, 4, 16, 1, false>(in, oref1, H, W, fp); run<FM, 2, 4, 16, 1, true>(in, o1, H, W, fp); diff("focal.mean f32");
    auto diffh = [&](const char *name) {
        cudaMemset(cnt, 0, 8);
        count_diff<<<132 * 8, 256>>>((const unsigned *)o[0], (const unsigned *)oref, n, cnt);
        unsigned long long h = 0;
        cudaMemcpy(&h, cnt, 8, cudaMemcpyDeviceToHost);
        printf("16-byte vs 32-byte halo,   %-14s: %llu cells differ (%s)\n", name, h, cudaGetErrorString(cudaGetLastError()));
        fflush(stdout);
    };
    cudaMemset(o[0], 0xff, n * 4); cudaMemset(oref, 0, n * 4);
    run<SlopeSqOp, 4, 3, 16, 1, true, 4>(in, oref1, H, W, sp); run<SlopeSqOp, 4, 3, 16, 1, true, 8>(in, o1, H, W, sp); diffh("slope(square)");
    run<HillshadeOp, 4, 3, 16, 1, true, 4>(in, oref1, H, W, hp); run<HillshadeOp, 4, 3, 16, 1, true, 8>(in, o1, H, W, hp); diffh("hillshade");
    run<FM, 4, 3, 16, 1, true, 4>(in, oref1, H, W, fp); run<FM, 4, 3, 16, 1, true, 8>(in, o1, H, W, fp); diffh("focal.mean f32");
    smi.stop();
    return 0;
}

"""Time the classify functions on a device-resident float32 DEM: one JSON line per function.

Each line records the card and its power limit (read in the same run) and:
* ms: the public function end to end on a device tensor, CUDA events around the call (median of --steps calls
  after --warmup), host work between its device passes included;
* gcells_s: cells per second of that call;
* bytes_per_cell: the algorithmic traffic -- 8 B for the per-cell pass (4 B read, 4 B written), 4 B for each
  order-statistic digit pass or moments pass over the raster, counted from the passes the call made; for
  maximum_breaks also the sort (4 B read and 4 B written to compact the finite keys, 12 B per digit pass) and
  4 B per pass over the sorted keys;
* hbm_fraction: bytes_per_cell x cells / ms over the H100 SXM data-sheet 3.35 TB/s.
natural_breaks has two lines: k = 5 with the default 20,000-cell sample of the whole DEM, and every cell
(num_sample=None) of a --nb-size square raster cut from it, small enough for the O(n^2) Jenks program.  Its
bytes_per_cell and hbm_fraction are null: the sample's stream and first-hit array are not raster passes.
One more line times ndvi, a band index with no halo (12 B per cell), for comparison with the per-cell pass.

--profile adds, per function, the device time of each kernel over one call from torch.profiler, taken after
the timed calls; for natural_breaks also the device time of its phases: the jump and generation of the word
stream, the resolve rounds, the first-hit pass and chains (with the compaction), the gather and sort of the
sample, the Jenks column passes, the per-cell pass, and the rest (the max pass).

Usage:  python scripts/bench_classify.py [--size 32768] [--nb-size 128] [--steps 5] [--warmup 2] [--profile]
"""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM = 3.35e12


def card():
    import torch
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
    except Exception:   # nvidia-smi missing: name from torch, power unknown
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


class Passes:
    """Counts the raster-sized passes the classify module makes, by wrapping its device calls."""

    def __init__(self, cl):
        self.bytes = 0
        self.cl = cl
        R = cl._Raster
        orig_select, orig_moments, orig_sort = R._select, R.moments, R.sorted_keys
        me = self

        def select(r, source, ptr, H, W, bits, ranks, hist0, tie=0):
            me.bytes += 4 * (1 if len(ranks) == 0 else bits // 8 - 1)
            return orig_select(r, source, ptr, H, W, bits, ranks, hist0, tie)

        def moments(r, above=float("-inf")):
            me.bytes += 4
            return orig_moments(r, above)

        def sorted_keys(r):
            me.bytes += 8 + 12 * cl._KEY_BITS.get(r.cells, 32) // 8
            return orig_sort(r)

        R._select, R.moments, R.sorted_keys = select, moments, sorted_keys


NB_PHASES = [("jump_and_generation", ("nb_seed_kernel", "nb_jump_kernel", "nb_gen_kernel")),
             ("resolve", ("nb_resolve_kernel<true>", "nb_starts_kernel")),
             ("first_hit_and_chains", ("nb_resolve_kernel<false>", "nb_chains_kernel", "nb_bitcount_kernel",
                                       "nb_block_scan_kernel", "nb_compact_kernel", "Memset")),
             ("gather_and_sort", ("index", "Index", "compact_keys_kernel", "sort_hist_kernel", "sort_scan_kernel",
                                  "sort_scatter_kernel", "Memcpy")),
             ("jenks", ("nb_jenks",)),
             ("per_cell", ("classify_cells_kernel",))]


def phase_of(key):
    for phase, marks in NB_PHASES:
        if any(m in key for m in marks):
            return phase
    return "other"


def time_ms(fn, steps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=32768)
    ap.add_argument("--nb-size", type=int, default=128)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    import ctypes

    import torch

    import xrspatial_b200 as xb
    from xrspatial_b200 import _lib
    from xrspatial_b200 import classify as cl
    if not torch.cuda.is_available():
        raise SystemExit("bench_classify needs a CUDA device")
    name, power = card()
    n = a.size
    dem = torch.empty((n, n), dtype=torch.float32, device="cuda")
    _lib.call("xrs_synth_terrain_f32", ctypes.c_void_p(dem.data_ptr()), n * 4, n, n, 0, 0, 7, 0.0, 3000.0,
              ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    agg = xb.DataArray(dem, dims=("y", "x"))
    cells = n * n
    passes = Passes(cl)
    runs = [("reclassify", lambda: xb.reclassify(agg, [500, 1000, 1500, 2000, 3000], [1, 2, 3, 4, 5])),
            ("binary", lambda: xb.binary(agg, [1000.0, 2000.0])),
            ("quantile", lambda: xb.quantile(agg, 10)),
            ("percentiles", lambda: xb.percentiles(agg)),
            ("box_plot", lambda: xb.box_plot(agg)),
            ("equal_interval", lambda: xb.equal_interval(agg, 5)),
            ("std_mean", lambda: xb.std_mean(agg)),
            ("head_tail_breaks", lambda: xb.head_tail_breaks(agg)),
            ("maximum_breaks", lambda: xb.maximum_breaks(agg, 5))]
    m = min(a.nb_size, n)
    small = xb.DataArray(dem[:m, :m].contiguous(), dims=("y", "x"))
    nb_runs = [("natural_breaks", n, lambda: xb.natural_breaks(agg, k=5)),
               ("natural_breaks num_sample=None", m, lambda: xb.natural_breaks(small, num_sample=None, k=5))]
    warnings.simplefilter("ignore")   # natural_breaks warns above 40,000 sampled cells
    for fn, f in runs:
        passes.bytes = 0
        f()
        per_cell = passes.bytes + 8
        ms = time_ms(f, a.steps, a.warmup)
        print(json.dumps({"fn": fn, "size": n, "dtype": "float32", "ms": round(ms, 3),
                          "gcells_s": round(cells / ms / 1e6, 2), "bytes_per_cell": per_cell,
                          "hbm_fraction": round(per_cell * cells / (ms * 1e-3) / HBM, 3),
                          "card": name, "power_limit": power}), flush=True)
    for fn, size, f in nb_runs:
        ms = time_ms(f, a.steps, a.warmup)
        print(json.dumps({"fn": fn, "size": size, "dtype": "float32", "ms": round(ms, 3),
                          "gcells_s": round(size * size / ms / 1e6, 2), "bytes_per_cell": None,
                          "hbm_fraction": None, "card": name, "power_limit": power}), flush=True)
    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        for fn, f in runs:
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                f()
                torch.cuda.synchronize()
            kernels = {}
            for e in prof.key_averages():
                if e.device_time_total > 0:
                    m = re.search(r"(\w+_kernel)", e.key)
                    k = m.group(1) if m else e.key[:40]
                    kernels[k] = round(kernels.get(k, 0.0) + e.device_time_total / 1000.0, 3)
            print(json.dumps({"fn": fn, "profile_ms": kernels}), flush=True)
        for fn, _, f in nb_runs:
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                f()
                torch.cuda.synchronize()
            phases = {}
            for e in prof.key_averages():
                if e.device_time_total > 0:
                    p = phase_of(e.key)
                    phases[p] = round(phases.get(p, 0.0) + e.device_time_total / 1000.0, 3)
            print(json.dumps({"fn": fn, "phases_ms": phases}), flush=True)
    torch.cuda.empty_cache()
    nir = agg
    red = xb.DataArray(dem.flip(0).contiguous(), dims=("y", "x"))
    ms = time_ms(lambda: xb.ndvi(nir, red), a.steps, a.warmup)
    print(json.dumps({"fn": "ndvi (band index, for comparison)", "size": n, "dtype": "float32", "ms": round(ms, 3),
                      "gcells_s": round(cells / ms / 1e6, 2), "bytes_per_cell": 12,
                      "hbm_fraction": round(12 * cells / (ms * 1e-3) / HBM, 3), "card": name,
                      "power_limit": power}), flush=True)


if __name__ == "__main__":
    main()

"""Time perlin and generate_terrain on the GPU: one JSON line per (function, size), float32 device rasters.

Each line records the card and its power limit (read in the same run), and in ms:
* tables: the device permutation tables (1 for perlin, 16 for generate_terrain), host clock around the call,
  which synchronizes;
* colrow / cell / epilogue: the column and row pass, the cell kernel, and the min/max reduction plus the
  normalising epilogue, from torch.profiler in a separate call;
* call: the public function end to end on a device tensor (median of --steps calls after --warmup);
and the float64 operations per cell the cell kernel executes, counted from noise_octave.cuh.  One more line
times RandomState(s).permutation(2**20) on this host (median of 5) for comparison with the device tables.
--reference-cpu also times the unmodified reference's _terrain_numpy on this host (needs XRS_REFERENCE_ROOT;
for scale only).

Usage:  python scripts/bench_terrain.py [--steps 3] [--warmup 1] [--sizes 4096 16384 32768]
"""
import argparse
import importlib
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# float64 operations of one octave at one cell (octave() in noise_octave.cuh): 4 gradients of 2 multiplies and 1
# add, the 2 distinct offsets xf - 1 and yf - 1, 3 lerps of a subtract, a multiply and an add
OCTAVE_OPS = 4 * 3 + 2 + 3 * 3
# terrain per octave adds a m to the running sum (a multiply and an add), then the cube's 2 multiplies
OPS = {"perlin": OCTAVE_OPS, "generate_terrain": 16 * (OCTAVE_OPS + 2) + 2}
STAGES = {"colrow": ("nz_col_kernel", "nz_row_kernel", "nz_stats_init_kernel"), "cell": ("nz_cell_kernel",),
          "epilogue": ("nz_minmax_kernel", "nz_epilogue_kernel")}


def card():
    import torch
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
    except Exception:   # nvidia-smi missing: name from torch, power unknown
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def call(fn, z):
    import xrspatial_b200 as xb
    agg = xb.DataArray(z, dims=("y", "x"))
    return xb.perlin(agg) if fn == "perlin" else xb.generate_terrain(agg)


def stage_ms(fn, z):
    import torch
    from torch.profiler import ProfilerActivity, profile
    call(fn, z)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call(fn, z)
        torch.cuda.synchronize()
    out = {k: 0.0 for k in STAGES}
    for e in prof.key_averages():
        for k, names in STAGES.items():
            if any(n in e.key for n in names):
                out[k] += e.device_time_total / 1000.0
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sizes", type=int, nargs="+", default=[4096, 16384, 32768])
    ap.add_argument("--reference-cpu", action="store_true")
    a = ap.parse_args()
    import torch
    pm = importlib.import_module("xrspatial_b200.perlin")
    name, power = card()
    host = []
    for s in range(5):
        t0 = time.perf_counter()
        np.random.RandomState(10 + s).permutation(2 ** 20)
        host.append((time.perf_counter() - t0) * 1e3)
    print(json.dumps({"what": "host RandomState.permutation(2**20)", "ms": round(statistics.median(host), 2),
                      "card": name, "power_limit": power}), flush=True)
    for fn, nseeds in (("perlin", 1), ("generate_terrain", 16)):
        seeds = list(range(10, 10 + nseeds))
        for _ in range(a.warmup):
            pm.perm_tables(seeds, "cuda")
        tt, rounds = [], []
        for _ in range(max(a.steps, 3)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pm.perm_tables(seeds, "cuda", rounds)
            torch.cuda.synchronize()
            tt.append((time.perf_counter() - t0) * 1e3)
        for n in a.sizes:
            z = torch.zeros((n, n), dtype=torch.float32, device="cuda")
            for _ in range(a.warmup):
                call(fn, z)
            times = []
            for _ in range(a.steps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                call(fn, z)
                torch.cuda.synchronize()
                times.append((time.perf_counter() - t0) * 1e3)
            st = stage_ms(fn, z)
            print(json.dumps({"fn": fn, "size": n, "dtype": "float32", "tables_ms": round(statistics.median(tt), 2),
                              "tables": nseeds, "shuffle_rounds": rounds[-1],
                              **{k + "_ms": round(v, 2) for k, v in st.items()},
                              "call_ms": round(statistics.median(times), 2),
                              "f64_ops_per_cell": OPS[fn], "card": name, "power_limit": power}), flush=True)
            del z
            torch.cuda.empty_cache()
    if a.reference_cpu:
        sys.path.insert(0, os.path.join(ROOT, "oracle"))
        import make_golden_terrain
        _, ter = make_golden_terrain._modules()
        for n in (50, 1024):
            t0 = time.perf_counter()
            ter._terrain_numpy(np.zeros((n, n), np.float32), 10, (0.0, 1.0), (0.0, 1.0), 4000)
            print(json.dumps({"what": "reference _terrain_numpy on this host", "size": n,
                              "ms": round((time.perf_counter() - t0) * 1e3, 1)}), flush=True)


if __name__ == "__main__":
    main()

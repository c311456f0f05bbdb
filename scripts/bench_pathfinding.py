"""Time a_star_search on the GPU: one JSON line per (workload, size, placement).

Workloads, each with 8-connectivity:
* open: no barriers; rand10 / rand30: 10 % and 30 % random barrier cells;
* dem: the synthetic generator's terrain (xrs_synth_terrain_f32, 0-4000 m) with every cell below 800 m NaN water;
* maze: a serpentine whose walls span every fourth row with a gap at alternating ends, so the path crosses the
  raster width once per two rows.  Its path has about H W / 4 cells and every corridor crosses W / 32 tiles, so
  its relaxation rounds grow with H W / 128: it is run at 1024^2 and 2048^2 only.
Placements: corner (start at the south-west corner, goal at the north-east) and near (goal 100 rows and 60
columns from a start at the centre).

The search fills the whole field of lengths to the goal whatever the placement (tiles are not pruned), so the
near placement shows that cost.  Each line records the card and its power limit, the median of --steps timed
calls of the public function on device tensors (CUDA events, after --warmup calls), the relaxation rounds and
the path length.  --profile adds the kernel split from torch.profiler in a separate call.  --reference times the
unmodified reference on a CPU host at <= 400^2 (needs XRS_REFERENCE_ROOT; for scale only).

Usage:  python scripts/bench_pathfinding.py [--steps 3] [--warmup 1] [--sizes 1024 4096 8192 16384] [--profile]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
    except Exception:   # nvidia-smi missing: name from torch, power unknown
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def raster(kind, n):
    """(cells, barriers) on the device as float32."""
    import torch
    from xrspatial_b200 import _lib
    if kind == "open":
        return torch.zeros((n, n), dtype=torch.float32, device="cuda"), []
    if kind.startswith("rand"):
        g = torch.Generator(device="cuda").manual_seed(7)
        dens = int(kind[4:]) / 100.0
        return (torch.rand((n, n), generator=g, device="cuda") < dens).float(), [1]
    if kind == "dem":
        t = torch.empty((n, n), dtype=torch.float32, device="cuda")
        _lib.call("xrs_synth_terrain_f32", ctypes.c_void_p(t.data_ptr()), n * 4, n, n, 0, 0, 1235, 0.0, 4000.0,
                  None)
        t[t < 800.0] = float("nan")
        return t, []
    z = torch.zeros((n, n), dtype=torch.float32, device="cuda")
    for i, r in enumerate(range(2, n - 1, 4)):
        z[r, :] = 1
        z[r, (n - 2, n - 1) if i % 2 == 0 else (0, 1)] = 0
    return z, [1]


def placement(where, n):
    if where == "corner":
        return (n - 1, 0), (0, n - 1)
    c = n // 2
    return (c, c), (c + 100, c + 60)


def rounds_of(z, bars, s, g):
    """The relaxation rounds of one search, from the C entry point."""
    import torch
    from xrspatial_b200 import _lib
    H, W = z.shape
    b = torch.as_tensor(np.append(np.asarray(bars, np.float64), 0.0), device="cuda")
    need = ctypes.c_int64()
    _lib.call("xrs_a_star_scratch_bytes", H, W, ctypes.byref(need))
    scr = torch.empty(need.value, dtype=torch.uint8, device="cuda")
    out = torch.empty((H, W), dtype=torch.float64, device="cuda")
    r = ctypes.c_int64()
    _lib.call("xrs_a_star_search", ctypes.c_void_p(z.data_ptr()), 0, W * 4, H, W, ctypes.c_void_p(b.data_ptr()),
              len(bars), 8, s[0], s[1], g[0], g[1], ctypes.c_void_p(out.data_ptr()), W * 8,
              ctypes.c_void_p(scr.data_ptr()), need.value, ctypes.byref(r), None)
    torch.cuda.synchronize()
    return r.value


def timed(fn, steps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def kernel_split(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    split = {}
    for e in prof.key_averages():
        for k in ("pf_mask_kernel", "pf_relax_kernel", "pf_fill_nan_kernel", "pf_walk_kernel"):
            if k in e.key:
                split[k] = split.get(k, 0.0) + e.device_time_total / 1e3
    return split


def reference_times():
    """The unmodified reference's a_star_search on this host (CPU), 10 % random barriers, corner to corner."""
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import make_golden_pathfinding as mg
    for n in (100, 200, 400):
        rng = np.random.default_rng(3)
        z = (rng.random((n, n)) < 0.1).astype(np.int64)
        z[n - 1, 0] = z[0, n - 1] = 0
        pts = mg.point(n, n, 1.0, 1.0, (n - 1, 0)), mg.point(n, n, 1.0, 1.0, (0, n - 1))
        mg.run(z, 1.0, 1.0, True, *pts, [1], 8, False, False)   # JIT warm-up
        t = time.perf_counter()
        out, _ = mg.run(z, 1.0, 1.0, True, *pts, [1], 8, False, False)
        print(json.dumps({"op": "a_star_search", "impl": "reference (CPU)", "workload": "rand10",
                          "shape": [n, n], "s": round(time.perf_counter() - t, 3),
                          "path_cells": int((~np.isnan(out)).sum())}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sizes", type=int, nargs="+", default=[1024, 4096, 8192, 16384])
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--reference", action="store_true")
    a = ap.parse_args()
    if a.reference:
        reference_times()
        return
    import torch
    import xrspatial_b200 as xb
    name, power = card()
    for n in a.sizes:
        for kind in ("open", "rand10", "rand30", "dem", "maze"):
            if kind == "maze" and n > 2048:
                continue
            z, bars = raster(kind, n)
            xs = np.arange(n, dtype=np.float64)
            da = xb.DataArray(z, dims=("y", "x"), coords={"y": xs[::-1].copy(), "x": xs}, attrs={"res": (1.0, 1.0)})
            for where in ("corner", "near"):
                s, g = placement(where, n)
                for cell in (s, g):
                    z[cell] = 0.0 if kind != "dem" else 1000.0
                call = lambda: xb.a_star_search(da, (float(n - 1 - s[0]), float(s[1])),   # noqa: E731
                                                (float(n - 1 - g[0]), float(g[1])), bars)
                out = call().data
                ms = timed(call, a.steps, a.warmup)
                path = out[~torch.isnan(out)]
                rec = {"op": "a_star_search", "workload": kind, "shape": [n, n], "placement": where,
                       "ms": round(ms, 3), "rounds": rounds_of(z, bars, s, g), "path_cells": int(path.numel()),
                       "path_length": float(path.max()) if path.numel() else None,
                       "gpu": name, "power_limit": power, "steps": a.steps}
                if a.profile:
                    rec["kernel_ms"] = {k: round(v, 3) for k, v in kernel_split(call).items()}
                print(json.dumps(rec), flush=True)
                del out, path
            del z, da
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

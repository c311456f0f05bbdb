"""Time viewshed on the GPU: one JSON line per (shape, observer).

* The reference benchmark's shapes (benchmarks/benchmarks/viewshed.py): nx in {100, 300, 1000, 3000},
  ny = nx / 2, its Gaussian bump with noise on linspace(-180, 180) x linspace(-90, 90), the observer at
  x=100, y=50 with observer_elev=1.
* 8192^2 and 16384^2 DEMs from the synthetic generator (xrs_synth_terrain_f32, 0-4000 m on 30 m cells), the
  observer 10 m (little is visible: most rays stop at their first ridge) and 1000 m (most rays run their whole
  length) above the centre cell and above a corner cell.

The work grows with H * W times the ray length, so each line records the card, its power limit, the median of
--steps timed calls (CUDA events around the public call on device tensors, after --warmup calls), cells/s and
the share of visible cells.  --profile adds, per shape, the time of the node pass and of the visibility pass from
torch.profiler in a separate call.

Usage:  python scripts/bench_viewshed.py [--steps 3] [--warmup 1] [--quick] [--profile]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import xrspatial_b200 as xb  # noqa: E402
from xrspatial_b200 import _lib  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
    except Exception:   # nvidia-smi missing: name from torch, power unknown
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def reference_dem(nx):
    """benchmarks/benchmarks/common.py get_xr_dataarray((nx // 2, nx), 'numpy')."""
    ny = nx // 2
    x = np.linspace(-180, 180, nx)
    y = np.linspace(-90, 90, ny)
    x2, y2 = np.meshgrid(x, y)
    rng = np.random.default_rng(71942)
    z = 100.0 * np.exp(-x2 ** 2 / 5e5 - y2 ** 2 / 2e5) + rng.normal(0.0, 2.0, (ny, nx))
    return torch.as_tensor(z, device="cuda"), x, y


def synth_dem(n):
    t = torch.empty((n, n), dtype=torch.float32, device="cuda")
    _lib.call("xrs_synth_terrain_f32", ctypes.c_void_p(t.data_ptr()), n * 4, n, n, 0, 0, 1235, 0.0, 4000.0, None)
    torch.cuda.synchronize()
    xs = np.arange(n) * 30.0
    return t, xs, xs[::-1].copy()


def timed(fn, steps, warmup):
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
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    split = {}
    for e in prof.key_averages():
        for k in ("vs_node_kernel", "vs_visibility_kernel"):
            if k in e.key:
                split[k] = split.get(k, 0.0) + e.device_time_total / 1e3
    return split


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--quick", action="store_true", help="the reference shapes and 8192^2 only")
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    name, power = card()
    runs = [("reference", nx, None, 1.0) for nx in (100, 300, 1000, 3000)]
    for n in (8192,) if a.quick else (8192, 16384):
        runs += [("synth", n, where, obs) for obs in (10.0, 1000.0) for where in ("centre", "corner")]
    for kind, n, where, obs in runs:
        if kind == "reference":
            z, xs, ys = reference_dem(n)
            x, y = 100, 50
        else:
            z, xs, ys = synth_dem(n)
            k = n // 2 if where == "centre" else 0
            x, y = xs[k], ys[k]
        da = xb.DataArray(z, dims=("y", "x"), coords={"y": ys, "x": xs})
        call = lambda: xb.viewshed(da, x=x, y=y, observer_elev=obs)   # noqa: E731
        out = call().data
        ms = timed(call, a.steps, a.warmup)
        H, W = z.shape
        rec = {"op": "viewshed", "dem": kind, "shape": [H, W], "observer": where or "x=100,y=50", "observer_elev": obs,
               "ms": round(ms, 3), "cells_per_s": H * W / (ms / 1e3), "visible": float((out >= 0).double().mean()),
               "gpu": name, "power_limit": power, "steps": a.steps}
        if a.profile:
            rec["kernel_ms"] = {k: round(v, 3) for k, v in kernel_split(call).items()}
        print(json.dumps(rec), flush=True)
        del z, da, out
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

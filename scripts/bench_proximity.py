"""Time proximity / allocation / direction on the GPU: one JSON line per (shape, target density, metric, mode).

Shapes 8192^2, 32768^2 and a narrow 32768 x 2048; target densities of one cell, 1e-4, 1e-2 and 30 % (a "water"
mask); every metric in distance mode, and every mode at 32768^2.  Each line records the card, its power limit,
the median of --runs timed calls (CUDA events, after warm-ups), Gcells/s and the rate over the 8 B/cell the
transform needs at least (read a 4-byte cell, write a 4-byte result).  At 8192^2 the Euclidean distance is also
compared with scipy.ndimage.distance_transform_edt when SciPy imports.

Usage:  python scripts/bench_proximity.py [--runs 20] [--quick]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import xrspatial_b200 as xb  # noqa: E402

px = importlib.import_module("xrspatial_b200.proximity")
ALGO_BYTES = 8


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
    except Exception:   # nvidia-smi missing: name from torch, power unknown
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def targets(H, W, density, rng):
    z = torch.zeros((H, W), dtype=torch.float32, device="cuda")
    if density == "one":
        z[H // 3, W // 5] = 1.0
    else:
        z = (torch.rand((H, W), device="cuda", generator=rng) < density).float()
    return z


def timed(fn, runs, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(runs):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=20)
    ap.add_argument("--quick", action="store_true", help="8192^2 only")
    args = ap.parse_args()
    name, power = card()
    rng = torch.Generator(device="cuda")
    rng.manual_seed(0)
    shapes = [(8192, 8192)] if args.quick else [(8192, 8192), (32768, 2048), (32768, 32768)]
    for H, W in shapes:
        xs, ys = np.arange(W) * 30.0, np.arange(H)[::-1] * 30.0
        ll_x, ll_y = np.linspace(-179.9, 179.9, W), np.linspace(80, -80, H)
        for density in ("one", 1e-4, 1e-2, 0.3):
            z = targets(H, W, density, rng)
            runs = [(m, "proximity") for m in ("EUCLIDEAN", "MANHATTAN", "GREAT_CIRCLE")]
            if H == W == 32768:
                runs += [("EUCLIDEAN", "allocation"), ("EUCLIDEAN", "direction")]
            for metric, mode in runs:
                gc = metric == "GREAT_CIRCLE"
                agg = xb.DataArray(z, dims=("y", "x"), coords={"y": ll_y if gc else ys, "x": ll_x if gc else xs})
                m = dict(proximity=0, allocation=1, direction=2)[mode]
                ms = timed(lambda: px._process(agg, "x", "y", [], np.inf, metric, m), args.runs)
                line = dict(op=mode, metric=metric, H=H, W=W, density=density, ms=round(ms, 3),
                            gcells_s=round(H * W / ms / 1e6, 2), algo_gb_s=round(H * W * ALGO_BYTES / ms / 1e6, 1),
                            card=name, power_limit=power, runs=args.runs)
                if H == W == 8192 and metric == "EUCLIDEAN" and density != "one":
                    try:
                        from scipy import ndimage
                        got = px._process(agg, "x", "y", [], np.inf, metric, 0).cpu().numpy()
                        edt = ndimage.distance_transform_edt(z.cpu().numpy() == 0, sampling=(30.0, 30.0))
                        want = np.sqrt((edt.astype(np.float32) ** 2).astype(np.float64)).astype(np.float32)
                        line["scipy_max_ulps"] = float((np.abs(got - want) / np.spacing(np.maximum(want, 1))).max())
                    except ImportError:
                        line["scipy_max_ulps"] = None
                print(json.dumps(line), flush=True)
            del z
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

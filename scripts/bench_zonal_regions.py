"""Time zonal regions (n = 4 and 8), trim and crop on device-resident float32 DEMs quantised into a few hundred
levels: one JSON line per (size, function).

Each line records the card and its power limit (read in the same run) and:
* ms: the public function end to end on a device tensor, CUDA events around the call (median of --steps calls
  after --warmup); for trim and crop that includes reading the four bounds back to the host;
* gcells_s: cells per second of that call;
* regions also reports how many regions the DEM has; trim and crop report read_gb_s (4 B read per cell over ms)
  and copy_fraction: that rate over the rate of a device-to-device copy of the same raster (read plus write
  bytes over the copy's time), measured in the same run.

trim is given values that no cell holds, so every cell is read and the bounds are the whole raster; crop is given
one level that lies in the DEM's middle rows.

Usage:  python scripts/bench_zonal_regions.py [--sizes 8192 32768] [--steps 5] [--warmup 2] [--levels 300]
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

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


def timed(fn, steps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def dem(size, levels):
    """A synthetic fBm DEM from the library's generator, quantised to `levels` steps."""
    import torch
    import xrspatial_b200 as xb
    t = torch.empty((size, size), dtype=torch.float32, device="cuda")
    xb._lib.call("xrs_synth_terrain_f32", ctypes.c_void_p(t.data_ptr()), size * 4, size, size, 0, 0, 12345,
                 ctypes.c_float(0.0), ctypes.c_float(float(levels)), ctypes.c_void_p(0))
    torch.floor_(t)
    torch.cuda.synchronize()
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[8192, 32768])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--levels", type=int, default=300)
    args = ap.parse_args()
    import torch
    import xrspatial_b200 as xb
    name, power = card()
    for size in args.sizes:
        t = dem(size, args.levels)
        agg = xb.DataArray(t, dims=("y", "x"))
        cells = size * size
        dst = torch.empty_like(t)
        copy_ms = timed(lambda: dst.copy_(t), args.steps, args.warmup)
        del dst
        copy_rate = 2 * 4 * cells / copy_ms / 1e6   # GB/s
        base = dict(card=name, power_limit=power, size=size, levels=args.levels, copy_ms=round(copy_ms, 3),
                    copy_gb_s=round(copy_rate, 1))
        for n in (4, 8):
            ms = timed(lambda: xb.regions(agg, neighborhood=n), args.steps, args.warmup)
            out = xb.regions(agg, neighborhood=n).data
            count = int(torch.unique(out).numel())
            del out
            print(json.dumps(dict(base, fn="regions", neighborhood=n, ms=round(ms, 3),
                                  gcells_s=round(cells / ms / 1e6, 3), regions=count)), flush=True)
        mid = float(t[size // 2, size // 2].item())
        for fn, call in (("trim", lambda: xb.trim(agg, values=(-1.0,))),
                         ("crop", lambda: xb.crop(agg, agg, zones_ids=(mid,)))):
            ms = timed(call, args.steps, args.warmup)
            rate = 4 * cells / ms / 1e6
            print(json.dumps(dict(base, fn=fn, ms=round(ms, 3), gcells_s=round(cells / ms / 1e6, 3),
                                  read_gb_s=round(rate, 1), copy_fraction=round(rate / copy_rate, 3))), flush=True)
        del agg, t
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

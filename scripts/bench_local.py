"""Time the local functions on device-resident stacks: one JSON line per (function, K, size, cell type).

Each line records the card and its power limit (read in the same run) and:
* ms: the public function end to end on a Dataset of CUDA tensors, CUDA events around the call (median of --steps
  calls after --warmup); that includes reading the per-call flags back to the host, and for combine numbering the
  distinct tuples and building attrs['key'];
* gcells_s: cells per second of that call;
* gb_s: bytes the call must move per cell (K cells read, the ref cell read by the frequencies, popularity and rank,
  8 B written, and the kind byte popularity and rank write) over ms, and copy_fraction: that rate
  over the rate of a device-to-device copy of one float32 raster of the same size (read plus write bytes over the
  copy's time), measured in the same run.

The stacks hold integer values 0-15, so combine sees at most 16**K distinct tuples; combine runs at K = 4 only,
where its key (at most 65536 tuples) stays small enough to build on the host.  The ref variable (the
frequencies, popularity, rank) holds 1 .. K.  32768**2 runs at K = 4 only: twelve float32 layers of that size and
the result would not leave room on an 80 GB card.

Usage:  python scripts/bench_local.py [--sizes 8192 32768] [--steps 20] [--warmup 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FUNCS = [("cell_stats", f) for f in ("sum", "mean", "median", "min", "max", "std")] + [
    (f, None) for f in ("combine", "lesser_frequency", "equal_frequency", "greater_frequency", "lowest_position",
                        "highest_position", "popularity", "rank")]
REF = {"lesser_frequency", "equal_frequency", "greater_frequency", "popularity", "rank"}


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[8192, 32768])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    import xrspatial_b200 as xb
    name, power = card()
    g = torch.Generator(device="cuda")
    g.manual_seed(0)
    for size in args.sizes:
        src = torch.empty((size, size), dtype=torch.float32, device="cuda")
        dst = torch.empty_like(src)
        copy_ms = timed(lambda: dst.copy_(src), args.steps, args.warmup)
        copy_gb_s = 2 * src.numel() * 4 / copy_ms / 1e6
        del src, dst
        stacks = [("float32", 4), ("uint16", 4)] + ([("float32", 12)] if size <= 8192 else [])
        for cells, K in stacks:
            ds = {"v%d" % j: torch.randint(0, 16, (size, size), generator=g, device="cuda").to(getattr(torch, cells))
                  for j in range(K)}
            ds["ref"] = torch.randint(1, K + 1, (size, size), generator=g, device="cuda", dtype=torch.int32)
            raster = xb.Dataset(ds)
            data = ["v%d" % j for j in range(K)]
            for fn, func in FUNCS:
                if fn == "combine" and K != 4:
                    continue
                f = getattr(xb.local, fn)
                if fn == "cell_stats":
                    call = lambda f=f, func=func: f(raster, data, func)   # noqa: E731
                elif fn in REF:
                    call = lambda f=f: f(raster, "ref", data)   # noqa: E731
                else:
                    call = lambda f=f: f(raster, data)   # noqa: E731
                ms = timed(call, args.steps, args.warmup)
                torch.cuda.empty_cache()
                n = size * size
                moved = K * ds["v0"].element_size() + 8 + (ds["ref"].element_size() if fn in REF else 0) + \
                    (1 if fn in ("popularity", "rank") else 0)
                gb_s = n * moved / ms / 1e6
                print(json.dumps({"function": func or fn, "K": K, "size": size, "cells": cells, "ms": round(ms, 3),
                                  "gcells_s": round(n / ms / 1e6, 3), "gb_s": round(gb_s, 1),
                                  "copy_gb_s": round(copy_gb_s, 1), "copy_fraction": round(gb_s / copy_gb_s, 3),
                                  "card": name, "power_limit": power}), flush=True)
            del ds, raster
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

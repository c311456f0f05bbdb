"""Time convolve_2d and the focal statistics over windows on both sides of the 49 x 49 limit of the tiled kernels,
on a device-resident synthetic DEM, and time the CPU oracle on a small sample.

For each window: ms per call (median of CUDA-event timings), Gcells/s, and taps/s (cells x participating taps per
second: every tap for convolve, the ones of the mask for the focal statistics).  Convolve also reports its share
of the FP64 FMA rate at the SM clock read in the same run (64 DFMA / clock / SM).  The last lines compare the
cost per (cell x participating tap) at 51 x 51 (first wide window) with 49 x 49 (last tiled window).

    python scripts/bench_wide_windows.py [rows] [cols]
"""
import ctypes
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle")]
import oracle as o  # noqa: E402
import xrspatial_b200 as xb  # noqa: E402
from xrspatial_b200 import _lib, focal  # noqa: E402
from xrspatial_b200.convolution import convolve_2d  # noqa: E402

FIVE = ["mean", "sum", "min", "max", "range"]   # no var / std: one sweep
KINDS = {4: "tiled", 6: "fused", 7: "tiled", 11: "wide", 12: "wide", 13: "wide fused"}


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True).stdout.strip().split(", ")
    return {"name": out[0], "power_limit_w": float(out[1]), "sm_mhz": float(out[2]), "max_sm_mhz": float(out[3])}


def timeit(fn, n=5):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(n):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def circle(k):
    y, x = np.mgrid[:k, :k] - k // 2
    return (x * x + y * y <= (k // 2) ** 2).astype(np.float64)


def main():
    rows = int(sys.argv[1]) if len(sys.argv) > 1 else 8192
    cols = int(sys.argv[2]) if len(sys.argv) > 2 else 8192
    dem = torch.empty((rows, cols), dtype=torch.float32, device="cuda")
    _lib.call("xrs_synth_terrain_f32", ctypes.c_void_p(dem.data_ptr()), cols * 4, rows, cols, 0, 0, 1235, 0.0,
              4000.0, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    info = gpu_info()
    print("%s, power limit %.0f W, %d SMs, max SM clock %.0f MHz; DEM %d x %d float32"
          % (info["name"], info["power_limit_w"], n_sm, info["max_sm_mhz"], rows, cols), flush=True)
    rng = np.random.default_rng(7)
    cost = {}

    def report(what, k, taps, fn, h):
        sub = dem[:h]
        ms = timeit(lambda: fn(sub))
        clk = gpu_info()["sm_mhz"]          # read right after the timed calls
        kind = KINDS.get(xb._lib.lib().xrs_debug_last_used_tma(), "?")
        cells = sub.numel()
        tps = cells * taps / ms * 1e3
        line = "%-22s k=%3d %-10s %9.2f ms %8.2f Gcells/s %8.3f Ttaps/s  SM %4.0f MHz" % (
            what, k, kind, ms, cells / ms / 1e6, tps / 1e12, clk)
        if what == "convolve mixed":
            line += "  %.2f of FP64 FMA" % (tps / (64 * n_sm * clk * 1e6))
        print(line, flush=True)
        cost[(what, k)] = ms / (cells * taps)

    for k in (49, 51, 101, 201):
        h = rows if k <= 101 else rows // 2
        w = rng.standard_normal((k, k)) * 0.3
        report("convolve mixed", k, k * k, lambda a: convolve_2d(a, w), h)
        c = circle(k)
        taps = int(c.sum())
        agg = lambda a: xb.DataArray(a, dims=("y", "x"))  # noqa: E731
        report("focal.apply mean", k, taps, lambda a: focal.apply(agg(a), c, func="mean"), h)
        report("focal.apply max", k, taps, lambda a: focal.apply(agg(a), c, func="max"), h)
        report("focal_stats x7", k, taps, lambda a: focal.focal_stats(agg(a), c), h // 2)
        report("focal_stats x5", k, taps, lambda a: focal.focal_stats(agg(a), c, stats_funcs=FIVE), h // 2)

    print("\ncost per (cell x tap), 51 x 51 (wide) over 49 x 49 (tiled); at most 1.5:")
    for what in ("convolve mixed", "focal.apply mean", "focal.apply max", "focal_stats x7", "focal_stats x5"):
        r = cost[(what, 51)] / cost[(what, 49)]
        print("  %-18s %.3f%s" % (what, r, "" if what.startswith("focal_stats") else ("  ok" if r <= 1.5 else "  OVER")))

    sample = dem[:256, :256].cpu().numpy()
    nt = o.max_threads()
    print("\nCPU oracle, %d threads, 256 x 256 sample:" % nt)
    for what, fn, taps in (("convolve mixed 101", lambda: o.convolve_2d_fma(sample, rng.standard_normal((101, 101)),
                                                                           nthreads=nt), 101 * 101),
                           ("focal mean circle 101", lambda: o.focal_apply(sample, circle(101), "mean", nthreads=nt),
                            int(circle(101).sum()))):
        t0 = time.perf_counter()
        fn()
        s = time.perf_counter() - t0
        print("  %-22s %8.3f s %8.4f Gcells/s %8.3f Gtaps/s" % (what, s, sample.size / s / 1e9,
                                                                  sample.size * taps / s / 1e9))


if __name__ == "__main__":
    main()

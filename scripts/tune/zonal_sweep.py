"""The zonal kernels on one GPU: the (zone, value) pair histogram, the default zonal.stats call, the group-by
pass on block and on noisy zones, and the float64 two-pass statistics.
usage: zonal_sweep.py [side]  -> ms and fraction of the measured copy peak per kernel."""
import ctypes, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import torch
from xrspatial_b200 import _lib

side = int(sys.argv[1]) if len(sys.argv) > 1 else 32768
PEAK = 6569.6
t = torch.empty((side, side), dtype=torch.float32, device="cuda")
_lib.call("xrs_synth_terrain_f32", ctypes.c_void_p(t.data_ptr()), side * 4, side, side, 0, 0, 1235, 0.0, 4000.0,
          ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))

# the (zone, value) pair histogram behind `majority` / `crosstab`, and the default zonal.stats call
import time
import xrspatial_b200 as xb
from xrspatial_b200 import zonal as Z
yy = torch.arange(side, device="cuda", dtype=torch.int32)[:, None] // (side // 32)
xx = torch.arange(side, device="cuda", dtype=torch.int32)[None, :] // (side // 32)
zones = (yy * 32 + xx).contiguous()
cats = (t * (16.0 / 4000.0)).floor_().clamp_(0, 15)
for _ in range(2):
    Z.pair_counts(zones, cats)
torch.cuda.synchronize()
ts = []
for _ in range(5):
    t0 = time.perf_counter(); Z.pair_counts(zones, cats); torch.cuda.synchronize(); ts.append((time.perf_counter() - t0) * 1e3)
ms = sorted(ts)[2]
print("pair_counts (kernel + host pivot) wall: %.3f ms  frac %.3f" % (ms, side * side * 8 / ms / 1e6 / PEAK))
za, ca = xb.DataArray(zones, dims=("y", "x")), xb.DataArray(cats, dims=("y", "x"))
ts = []
for _ in range(4):
    t0 = time.perf_counter(); df = xb.zonal_stats(za, ca); torch.cuda.synchronize(); ts.append((time.perf_counter() - t0) * 1e3)
print("zonal.stats default list (incl. majority) wall: %.3f ms" % sorted(ts)[1])
print(df.head(3))

# zones with irregular outlines (contour bands of a second fBm surface): about every other warp-row holds a
# boundary cell, unlike the block zones of the benchmark
t2 = torch.empty((side, side), dtype=torch.float32, device="cuda")
_lib.call("xrs_synth_terrain_f32", ctypes.c_void_p(t2.data_ptr()), side * 4, side, side, 0, 0, 99, 0.0, 4000.0,
          ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
zirr = (t2 * (64.0 / 4000.0)).floor_().clamp_(0, 63).to(torch.int32)
del t2

for name, zz in (("block zones", zones), ("noisy zones (64 contour bands of a rough fBm surface)", zirr)):
    for _ in range(2):
        Z.hash_partials(zz, t)
    torch.cuda.synchronize()
    ts = []
    for _ in range(5):
        t0 = time.perf_counter(); Z.hash_partials(zz, t); torch.cuda.synchronize(); ts.append((time.perf_counter() - t0) * 1e3)
    ms = sorted(ts)[2]
    print("hash_partials, %s: %.3f ms  frac %.3f" % (name, ms, side * side * 8 / ms / 1e6 / PEAK))
t64 = t[: side // 2].to(torch.float64)
z64 = zones[: side // 2].contiguous()
a64, b64 = xb.DataArray(z64, dims=("y", "x")), xb.DataArray(t64, dims=("y", "x"))
ts = []
for _ in range(4):
    t0 = time.perf_counter(); df = xb.zonal_stats(a64, b64, stats_funcs=["mean", "std", "var", "count"]); torch.cuda.synchronize(); ts.append((time.perf_counter() - t0) * 1e3)
ms = sorted(ts)[1]
print("zonal.stats float64 values (two hash passes), %d x %d: %.3f ms  frac %.3f of 2 x 12 B/cell" %
      (side // 2, side, ms, (side // 2) * side * 24 / ms / 1e6 / PEAK))

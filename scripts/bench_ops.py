"""Per-operator device-resident throughput table (Mcells/s, GB/s of algorithmic bytes, fraction
of the HBM peak) for every kernel on the hot path, as JSON on stdout.  Not the headline benchmark
(bench.py).  usage: bench_ops.py [side] [reps]"""
import ctypes, json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import xrspatial_b200 as xb
from xrspatial_b200 import _lib, focal
from xrspatial_b200.convolution import convolve_2d

side = int(sys.argv[1]) if len(sys.argv) > 1 else 32768
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 10
peak = 3350.0   # H100 SXM data sheet
try:
    peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception:
    pass


def synth(seed, lo, hi, h=side, w=side):
    t = torch.empty((h, w), dtype=torch.float32, device="cuda")
    _lib.call("xrs_synth_terrain_f32", ctypes.c_void_p(t.data_ptr()), w * 4, h, w, 0, 0, seed, lo, hi,
              ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    return t


def timeit(fn, n=reps, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(n + 1)]
    ev[0].record()
    for i in range(n):
        fn()
        ev[i + 1].record()
    torch.cuda.synchronize()
    return float(np.median([ev[i].elapsed_time(ev[i + 1]) for i in range(n)]))


dem = synth(1235, 0.0, 4000.0)
agg = xb.DataArray(dem, dims=("y", "x"), attrs={"res": (30.0, 30.0)})
cells = side * side
rows = []


def add(name, ms, bytes_per_cell, ncells=cells, note=""):
    gbs = ncells * bytes_per_cell / (ms * 1e-3) / 1e9
    rows.append(dict(op=name, ms=ms, mcells_s=ncells / (ms * 1e-3) / 1e6, alg_bytes_per_cell=bytes_per_cell,
                     gbs=gbs, frac_of_measured_hbm=gbs / peak, note=note))
    print("%-28s %9.3f ms %12.0f Mcells/s %8.0f GB/s  %.3f" % (name, ms, rows[-1]["mcells_s"], gbs, gbs / peak), file=sys.stderr, flush=True)


add("slope", timeit(lambda: xb.slope(agg)), 8)
odd = xb.DataArray(dem[:, :side - 2], dims=("y", "x"), attrs={"res": (30.0, 30.0)})   # W % 4 != 0 -> direct-load kernel
add("slope, direct-load path (W-2)", timeit(lambda: xb.slope(odd)), 8, ncells=side * (side - 2))
i16 = xb.DataArray(dem.round().to(torch.int16), dims=("y", "x"), attrs={"res": (30.0, 30.0)})
add("slope, int16 DEM ingested directly", timeit(lambda: xb.slope(i16)), 6, note="2 B read + 4 B written per cell")
f64 = xb.DataArray(dem[: side // 2].to(torch.float64), dims=("y", "x"), attrs={"res": (30.0, 30.0)})
add("slope, float64 DEM ingested directly", timeit(lambda: xb.slope(f64)), 12, ncells=side * side // 2,
    note="8 B read + 4 B written per cell")
del i16, f64
from xrspatial_b200.slope import slope as _sl
lat = np.linspace(46.5, 40.0, side); lon = np.linspace(7.0, 13.5, side)
geo = xb.DataArray(dem[: side // 4], dims=("lat", "lon")); geo["lat"] = lat[: side // 4]; geo["lon"] = lon
add("slope geodesic (f32 elev, regular grid)", timeit(lambda: _sl(geo, method="geodesic"), n=3), 8, ncells=dem[: side // 4].numel(),
    note="FP64-bound: ~300 FP64 ops per cell")
add("aspect", timeit(lambda: xb.aspect(agg)), 8)
add("curvature", timeit(lambda: xb.curvature(agg)), 8)
add("hillshade", timeit(lambda: xb.hillshade(agg)), 8)
add("focal.mean f32", timeit(lambda: xb.mean(agg)), 8)
add("surface suite (4 outputs)", timeit(lambda: xb.surface_suite(agg)), 20)
add("suite slope+aspect+curvature", timeit(lambda: xb.surface_suite(agg, products=("slope", "aspect", "curvature"))), 16)
d64 = dem[: side // 2].to(torch.float64)
a64 = xb.DataArray(d64, dims=("y", "x"))
add("focal.mean f64", timeit(lambda: xb.mean(a64)), 16, ncells=d64.numel())
del d64, a64
for k in (3, 9, 25):
    kern = np.ones((k, k)) / (k * k)
    add("convolve_2d k=%d uniform (ones/k^2)" % k, timeit(lambda: convolve_2d(dem, kern), n=max(3, reps // 2)), 8,
        note="k=3: strip kernel; k>3: running-box kernel (box_stream.cu)")
krng = np.random.default_rng(7)
for k in (9, 25):
    kern = krng.standard_normal((k, k))
    sub = dem[: side // (2 if k == 9 else 8)]
    add("convolve_2d k=%d mixed weights" % k, timeit(lambda: convolve_2d(sub, kern), n=max(3, reps // 2)), 8,
        ncells=sub.numel(), note="f64 accumulate; bound = FP64 FMA rate (2*k*k flop/cell)")
k5 = np.ones((5, 5))
sub = dem[: side // 4]
sagg = xb.DataArray(sub, dims=("y", "x"))
add("focal.apply mean 5x5", timeit(lambda: focal.apply(sagg, k5), n=3), 8, ncells=sub.numel())
add("focal_stats 7 statistics 5x5 (fused)", timeit(lambda: focal.focal_stats(sagg, k5), n=3), 32, ncells=sub.numel(),
    note="one pass: tile loaded once, swept twice, 7 planes written in place")
nir, red, blue = synth(2001, 0.02, 0.6), synth(2002, 0.02, 0.6), synth(2003, 0.02, 0.6)
A = lambda t: xb.DataArray(t, dims=("y", "x"))  # noqa: E731
add("ndvi", timeit(lambda: xb.ndvi(A(nir), A(red))), 12)
add("savi", timeit(lambda: xb.savi(A(nir), A(red))), 12)
add("evi", timeit(lambda: xb.evi(A(nir), A(red), A(blue))), 16)
del nir, red, blue
yy = torch.arange(side, device="cuda", dtype=torch.int32)[:, None] // (side // 32)
xx = torch.arange(side, device="cuda", dtype=torch.int32)[None, :] // (side // 32)
zones = (yy * 32 + xx).contiguous()
zagg = A(zones)
add("zonal.stats 1024 block zones", timeit(lambda: xb.zonal_stats(zagg, agg), n=3), 8,
    note="includes zone-id discovery (min/max + presence pass) and host finalisation")
ids = list(range(1024))
from xrspatial_b200 import zonal as Z  # noqa: E402
zt, vt = zones, dem
sel = np.arange(1024, dtype=np.int32)
add("zonal hash partials (ids discovered)", timeit(lambda: Z.hash_partials(zt, vt)), 8,
    note="xrs_zonal_hash_run: pivot, accumulation, compaction + tiny D2H")
hz = ((torch.arange(side, device="cuda", dtype=torch.int64)[:, None] * 7919 +
       torch.arange(side, device="cuda", dtype=torch.int64)[None, :] * 104729) % 1024).to(torch.int32)
add("zonal hash partials, scattered zones", timeit(lambda: Z.hash_partials(hz, vt), n=3), 8,
    note="worst case: zone changes every cell")
# next-tier rows (SURVEY.md section 8f): hotspots, majority, crosstab
from xrspatial_b200.convolution import circle_kernel  # noqa: E402
hsub = xb.DataArray(dem[: side // 4], dims=("y", "x"))
ck = circle_kernel(1, 1, 2)
add("hotspots, circle kernel r=2 (5x5)", timeit(lambda: xb.hotspots(hsub, ck), n=3), 5, ncells=hsub.data.numel(),
    note="convolve + global mean/std + int8 classification")
cats = ((dem * (16.0 / 4000.0)).floor().clamp_(0, 15)).contiguous()
cagg = A(cats)
add("zonal.crosstab 1024 zones x 16 classes", timeit(lambda: xb.zonal_crosstab(zagg, cagg), n=3), 8,
    note="xrs_zonal_pair_count + host pivot")
add("zonal.stats majority, 16 classes", timeit(lambda: xb.zonal_stats(zagg, cagg, stats_funcs=["majority"]), n=3), 8,
    note="hash partials + pair histogram")
json.dump(dict(side=side, peak_gbs=peak, rows=rows), sys.stdout, indent=1)

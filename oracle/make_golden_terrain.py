"""Generate tests/golden/terrain_reference.npz and terrain_signature.json from the UNMODIFIED reference.

TEST INFRASTRUCTURE (needs a checkout of the reference, like make_golden.py; the existing golden files are not
touched).  Every output comes from the reference's NumPy path: `_perlin_numpy` (perlin.py:77) for perlin, and for
generate_terrain `_terrain_numpy` (terrain.py:64) at the ranges the reference's own `_scale` gives, plus
`_gen_terrain` (terrain.py:36) for the field before the cube: it divides its first argument in place before
`height_map ** 3` rebinds the name, so the array passed in ends up holding the field after / 1.97.  terrain.py
imports pandas and datashader at module level for its coordinates; neither is used on this seam, so both are
stubbed when missing.

* perlin: the docstring example (3 x 4 float32 zeros) and the reference tests' 50 x 50 float32 zeros, then seeded
  rasters of 1 x 1 .. 37 x 53 in float32 and float64 over the frequencies (1, 1), (3, 2.5), (0.5, 7), (-2, 3),
  (64, 64), (2^21, 1) and seeds 0, 5, 2^32 - 1, plus frequencies at which the reference raises IndexError (outer
  and inner indices of its doubled table).  A case that raised is stored with `raised` set and no output.
* terrain: the reference tests' 50 x 50 float32 zeros, the defaults at 256 x 300, seeds 0, 10 and 2^32 - 16,
  extents giving a sub-range, negative scaled coordinates and scaled coordinates above 1, float64 cells, negative
  cells (the sum starts from -0) and a raster holding one NaN.

Usage:  XRS_REFERENCE_ROOT=<reference checkout> python oracle/make_golden_terrain.py
"""
import inspect
import json
import os
import sys
import types
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_loader  # noqa: E402
from make_golden import encode_default  # noqa: E402

OUT_DIR = os.path.join(os.path.dirname(HERE), "tests", "golden")

PERLIN_SHAPES = [(1, 1), (1, 6), (5, 1), (3, 4), (8, 8), (13, 7), (37, 53)]
PERLIN_FREQS = [(1, 1), (3, 2.5), (0.5, 7), (-2, 3), (64, 64), (2 ** 21, 1)]
PERLIN_SEEDS = [0, 5, 2 ** 32 - 1]
# (shape, freq) pairs at which the table index leaves [-2^21, 2^21) for some or every seed
PERLIN_EDGES = [((3, 4), (2 ** 22, 1)), ((3, 4), (-(2 ** 21) - 8, 1)), ((2, 1), (1, 3 * 2 ** 20)),
                ((2, 3), (1, -3 * 2 ** 20)), ((4, 2), (2 ** 21 - 2, 2 ** 20)), ((1, 2), (2 ** 21 + 2, 1)),
                ((2, 2), (np.nan, 1)), ((2, 2), (1, np.inf)),
                # P[0], P[1] of seed 0 are 875681, 1046907: row 1 at yi = 1050244 reaches index 2^21 for seed 0 only
                ((2, 1), (1, 2 * 1050244)), ((2, 1), (1, 2 * 1050243))]


def _modules():
    for name in ("pandas",):
        if name not in sys.modules:
            try:
                __import__(name)
            except ImportError:
                sys.modules[name] = types.ModuleType(name)
    return ref_loader.load("perlin"), ref_loader.load("terrain")


def perlin_cases():
    cases = [((3, 4), (1, 1), 5, np.float32), ((50, 50), (1, 1), 5, np.float32)]
    for shape in PERLIN_SHAPES:
        for dt in (np.float32, np.float64):
            for freq in PERLIN_FREQS:
                for seed in PERLIN_SEEDS:
                    cases.append((shape, freq, seed, dt))
    for shape, freq in PERLIN_EDGES:
        for seed in (0, 5):
            cases.append((shape, freq, seed, np.float32))
    return cases


def terrain_cases():
    """(shape, dtype, x_range, y_range, seed, zfactor, full_extent, fill, nan_at)"""
    d = ((0, 500), (0, 500))
    return [
        ((50, 50), np.float32) + d + (10, 4000, None, 0.0, -1),
        ((256, 300), np.float32) + d + (10, 4000, None, 0.0, -1),
        ((40, 30), np.float32) + d + (0, 4000, None, 0.0, -1),
        ((40, 30), np.float32) + d + (2 ** 32 - 16, 4000, None, 0.0, -1),
        ((33, 47), np.float32, (100, 200), (50, 450), 10, 10, (0, 0, 500, 500), 0.0, -1),
        ((33, 47), np.float32, (-250, 250), (-100, 40), 3, 4000, (0, 0, 500, 500), 0.0, -1),
        ((33, 47), np.float32, (0, 1500), (400, 1300), 7, 1, (0, 0, 500, 500), 0.0, -1),
        ((48, 64), np.float64) + d + (10, 4000, None, 0.0, -1),
        ((31, 29), np.float64, (-20e6, 20e6), (-20e6, 20e6), 2, 10, (-40e6, -40e6, 40e6, 40e6), 0.0, -1),
        ((24, 36), np.float32) + d + (10, 4000, None, -1.5, -1),
        ((24, 36), np.float32) + d + (10, 4000, None, 0.0, 77),
    ]


def main():
    per, ter = _modules()
    np.seterr(all="ignore")
    warnings.simplefilter("ignore")
    pm, pf, po, pv = [], [], [0], []
    for (h, w), freq, seed, dt in perlin_cases():
        raised = 0
        try:
            out = per._perlin_numpy(np.zeros((h, w), dt), freq, seed)
            pv.append(out.astype(np.float64).ravel())
        except IndexError:
            raised = 1
        pm.append([h, w, dt == np.float64, seed, raised])
        pf.append(freq)
        po.append(po[-1] + (0 if raised else h * w))
    tm, tr, te, ts, to, tv, tp = [], [], [], [], [0], [], []
    for (h, w), dt, xr_, yr_, seed, zf, ext, fill, nan_at in terrain_cases():
        full = ext if ext is not None else (xr_[0], yr_[0], xr_[1], yr_[1])
        xs = (ter._scale(xr_[0], (full[0], full[2]), (0.0, 1.0)), ter._scale(xr_[1], (full[0], full[2]), (0.0, 1.0)))
        ys = (ter._scale(yr_[0], (full[1], full[3]), (0.0, 1.0)), ter._scale(yr_[1], (full[1], full[3]), (0.0, 1.0)))
        data = np.full((h, w), fill, dt)
        if nan_at >= 0:
            data.ravel()[nan_at] = np.nan
        out = ter._terrain_numpy(data.copy(), seed, xs, ys, zf)
        pre = data * 0
        ter._gen_terrain(pre, seed, x_range=xs, y_range=ys)
        tm.append([h, w, dt == np.float64, seed, zf, ext is not None, nan_at])
        tr.append(list(xr_) + list(yr_))
        te.append(list(ext) if ext is not None else [0, 0, 0, 0])
        ts.append(list(xs) + list(ys))
        tv.append(out.astype(np.float64).ravel())
        tp.append(pre.astype(np.float64).ravel())
        to.append(to[-1] + h * w)
    fills = np.array([c[7] for c in terrain_cases()])
    np.savez_compressed(
        os.path.join(OUT_DIR, "terrain_reference.npz"),
        perlin_meta=np.array(pm, np.int64), perlin_freq=np.array(pf, np.float64), perlin_off=np.array(po, np.int64),
        perlin_out=np.concatenate(pv), terrain_meta=np.array(tm, np.int64), terrain_ranges=np.array(tr, np.float64),
        terrain_extent=np.array(te, np.float64), terrain_scaled=np.array(ts, np.float64), terrain_fill=fills,
        terrain_off=np.array(to, np.int64), terrain_out=np.concatenate(tv), terrain_precube=np.concatenate(tp))
    sig = {}
    for mod, fn in ((per, "perlin"), (ter, "generate_terrain")):
        sig[fn] = [[k, encode_default(v.default)]
                   for k, v in inspect.signature(inspect.unwrap(getattr(mod, fn))).parameters.items()]
    with open(os.path.join(OUT_DIR, "terrain_signature.json"), "w") as f:
        json.dump(sig, f, indent=1, sort_keys=True)
    print("perlin cases %d (%d raised), terrain cases %d" % (len(pm), sum(m[4] for m in pm), len(tm)))


if __name__ == "__main__":
    main()

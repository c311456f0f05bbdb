"""Generate tests/golden/zonal_regions_reference.npz and zonal_regions_signature.json from the UNMODIFIED
reference.

TEST INFRASTRUCTURE (needs a checkout of the reference and numba, like make_golden.py; the existing golden files
are not touched).  Every label comes from the reference's own `_area_connectivity` (zonal.py:1406-1549) and every
bound from its `_trim` / `_crop` (zonal.py:1651-1940), run through numba.

* `reg{i}_in`, `reg{i}_out`, `reg_n[i]`: regions cases -- the docstring examples, the reference tests' fixtures,
  about 300 seeded rasters up to 64 x 64 (few values, near-ties at the tolerance, NaN and +-inf, large-magnitude
  and extreme integers of all eight integer types, 1 x N and N x 1; integer rasters small
  enough that every label fits the type), and a few rasters of 256-512 cells a side (`large_rasters`).
* `bnd{i}_in`, `bnd{i}_values`, `bnd{i}_mode` (0 trim, 1 crop), `bnd{i}_out` (top, bottom, left, right): bounds
  cases with int, float and NaN value lists, including ones where nothing qualifies.
* The JSON holds the public signatures and suggest_zonal_canvas / get_full_extent results.

Usage:  XRS_REFERENCE_ROOT=<reference checkout> python oracle/make_golden_zonal_regions.py
"""
import inspect
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_loader  # noqa: E402
from make_golden import encode_default  # noqa: E402

OUT_DIR = os.path.join(os.path.dirname(HERE), "tests", "golden")
INTS = ["int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64"]


def fixtures():
    doc4 = np.array([[1, 1, 0, 2, 2], [1, 1, 0, 2, 2], [0, 0, 0, 0, 0], [3, 3, 0, 3, 3], [3, 3, 0, 3, 3]], np.float64)
    doc8 = np.array([[1, 0, 1], [0, 1, 0], [1, 0, 1]], np.float64)
    t4 = np.array([[0, 0, 0, 0], [0, 4, 0, 0], [1, 4, 4, 0], [1, 1, 1, 0], [0, 0, 0, 0]])
    t8 = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1], [0, 0, 0, 1]])
    t4f, t8f = t4.astype(np.float64), t8.astype(np.float64)
    t4f[0, 3] = t8f[0, 3] = np.nan
    return [(doc4, 4), (doc8, 8), (t4.astype(np.int64), 4), (t4f, 4), (t8.astype(np.int64), 8), (t8f, 8)]


def seeded_raster(rng, i):
    H, W = (int(v) for v in rng.integers(1, 65, 2))
    if i % 10 == 0:
        H = 1
    elif i % 10 == 1:
        W = 1
    kind = i % 6
    dt = np.dtype(["float64", "float32"][i % 2] if kind < 3 else INTS[(i // 6) % 8])
    while dt.kind in "iu" and H * W > np.iinfo(dt).max:   # the reference's labels wrap past the type's range
        H, W = max(1, H // 2), max(1, W - W // 3)
    if kind == 0:    # few values, NaN and +-inf
        a = rng.integers(0, 3, (H, W)).astype(dt)
        a[rng.random((H, W)) < 0.1] = np.nan
        a[rng.random((H, W)) < 0.03] = np.inf
        a[rng.random((H, W)) < 0.03] = -np.inf
    elif kind == 1:  # near-ties at the tolerance: non-transitive chains
        base = [1.0, 1e3, 1e5, 0.0][i % 4]
        step = 1e-08 + 1e-05 * abs(base)
        a = (base + step * rng.integers(0, 4, (H, W)) * rng.choice([0.5, 0.999, 1.0, 1.001], (H, W))).astype(dt)
        a[rng.random((H, W)) < 0.05] = np.nan
    elif kind == 2:  # a smooth ramp quantised finely: long diagonal chains
        H, W = min(H, 24), min(W, 24)   # its floats do not compress
        y, x = np.mgrid[0:H, 0:W]
        a = ((y + x * 0.7) * 1e-5 * (1 + rng.random())).astype(dt)
    elif kind == 3:  # small integers
        a = rng.integers(0, 3, (H, W)).astype(dt)
    elif kind == 4:  # large magnitudes: neighbours within 1e-5 |c|
        info = np.iinfo(dt)
        base = int(info.max) // 2 if info.bits > 16 else int(info.max) - 40
        a = (base - rng.integers(0, 3, (H, W)) * max(1, base // 100000)).astype(dt)
    else:            # the type's extremes
        info = np.iinfo(dt)
        pool = np.array([info.min, info.min + 1, 0, 1, info.max - 1, info.max], dtype=dt)
        a = pool[rng.integers(0, len(pool), (H, W))]
    return np.ascontiguousarray(a)


def large_rasters(rng):
    """Rasters of 256-512 cells a side.  Random few-valued ones (many small regions, the reference's slowest input)
    are kept to 256 x 256 and below, because their labels do not compress; the larger ones are a quantised smooth
    field with large, winding regions and a serpentine band."""
    out = [(rng.integers(0, 3, (256, 256)).astype(np.float32), 8), (rng.integers(0, 2, (192, 192)).astype(np.float32), 4)]
    y, x = np.mgrid[0:512, 0:512]
    field = np.floor(6 * (np.sin(x / 23.0) * np.cos(y / 31.0) + 0.5 * np.sin((x + 2 * y) / 47.0)))
    out += [(field.astype(np.float32), 4), (np.ascontiguousarray(field[:, :320]), 8)]
    serp = ((y // 4) % 2 == 0) | ((y // 4 % 4 == 1) & (x == 511)) | ((y // 4 % 4 == 3) & (x == 0))
    out.append((serp.astype(np.int32), 4))
    return out


def bounds_cases(rng):
    cases = []
    t = np.array([[0, 0, 0, 0], [0, 4, 0, 0], [0, 4, 4, 0], [0, 1, 1, 0], [0, 0, 0, 0]], np.int64)
    c = np.array([[0, 4, 0, 3], [0, 4, 4, 3], [0, 1, 1, 3], [0, 1, 1, 0], [0, 0, 0, 0]], np.int64)
    cases += [(t, (0,), 0), (c, (1, 3), 1), (c, (0,), 1), (t, (7,), 1), (t, (0, 1, 4), 0), (t, (np.nan,), 0)]
    f = t.astype(np.float32)
    f[0, 0] = np.nan
    cases += [(f, (np.nan,), 0), (f, (0.0,), 0), (f + np.float32(0.1), (0.1,), 0), (f, (4.0,), 1),
              (np.full((1, 5), 2.0), (2.0,), 0), (np.full((4, 1), 2), (2,), 0), (np.full((3, 3), 2), (2,), 0),
              (np.array([[2 ** 53 + 1, 0], [0, 0]], np.int64), (float(2 ** 53),), 1),
              (np.array([[2 ** 53 + 1, 0], [0, 0]], np.int64), (2 ** 53,), 1)]
    for i in range(40):
        H, W = (int(v) for v in rng.integers(1, 40, 2))
        a = np.zeros((H, W), [np.float64, np.float32, np.int32, np.uint8][i % 4])
        r0, c0 = rng.integers(0, H), rng.integers(0, W)
        a[r0:r0 + rng.integers(1, 6), c0:c0 + rng.integers(1, 6)] = rng.integers(1, 4)
        vals = [(0,), (0.0,), (1, 2), (1.0, 2.0, 3.0), (5,), (np.nan, 0.0)][i % 6]
        cases.append((a, vals, i % 2))
    return cases


def main():
    z = ref_loader.load("zonal")
    rng = np.random.default_rng(20261018)
    out = {}
    regs = fixtures() + [(seeded_raster(rng, i), 4 + 4 * ((i // 48) % 2)) for i in range(300)] + large_rasters(rng)
    for i, (a, n) in enumerate(regs):
        out["reg%d_in" % i] = a
        out["reg%d_out" % i] = z._area_connectivity(a, n)
    out["reg_n"] = np.array([n for _, n in regs], np.int64)
    for i, (a, vals, mode) in enumerate(bounds_cases(rng)):
        fn = z._crop if mode else z._trim
        out["bnd%d_in" % i] = a
        out["bnd%d_values" % i] = np.array(vals, dtype=np.int64 if all(isinstance(v, int) for v in vals) else np.float64)
        out["bnd%d_mode" % i] = np.int64(mode)
        out["bnd%d_out" % i] = np.array(fn(a, vals), np.int64)
    np.savez_compressed(os.path.join(OUT_DIR, "zonal_regions_reference.npz"), **out)

    def params(f):
        return [[k, encode_default(v.default)] for k, v in inspect.signature(inspect.unwrap(f)).parameters.items()]
    canvas = []
    for args in ((2, (0, 20), (0, 10), "Geographic", 2), (2e9, (-1e6, 1e6), (0, 1e6), "Mercator", 20),
                 (1234.5, (-3e6, 7e6), (-1e5, 2.5e6), "Mercator", 25), (0.37, (-170, 33.3), (-80, 10), "Geographic", 7),
                 (5e8, (-20e6, 20e6), (-20e6, 20e6), "Mercator", 1)):
        canvas.append([list(args), list(z.suggest_zonal_canvas(*args))])
    sig = {"signatures": {f: params(getattr(z, f)) for f in ("regions", "trim", "crop", "suggest_zonal_canvas",
                                                           "get_full_extent")},
           "canvas": canvas,
           "full_extent": {c: [list(v) for v in z.get_full_extent(c)] for c in ("Mercator", "Geographic")}}
    with open(os.path.join(OUT_DIR, "zonal_regions_signature.json"), "w") as f:
        json.dump(sig, f, indent=1)
    print("%d regions cases, %d bounds cases" % (len(regs), len(bounds_cases(np.random.default_rng(0)))))


if __name__ == "__main__":
    main()

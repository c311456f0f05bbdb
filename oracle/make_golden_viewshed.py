"""Generate tests/golden/viewshed_reference.npz and viewshed_signature.json from the UNMODIFIED reference.

TEST INFRASTRUCTURE (needs a checkout of the reference, like make_golden.py; the existing golden files are not
touched).  Every output comes from the reference's own `_viewshed_cpu` (viewshed.py:1505-1586): the coordinate
checks, the nearest-coordinate pick, the event list, the lexsort and the red-black sweep.  ref_loader's stub
DataArray has no `indexes` / `sel`, so a small adapter supplies them with pandas' nearest lookup, the one xarray
uses.

* `doc_*`: the docstring example (viewshed.py:1623-1656).
* `tv_*`: the reference test's 5 x 5 fixture (test_viewshed.py `empty_agg`: datashader pixel centres of
  (-20, 20)^2, int64 cells) for every observer position, observer elevation and elevation under the observer
  that `test_viewshed` loops over; `flat_*`: `test_viewshed_flat`'s four parameter sets.
* `small_*`: seeded rasters of 3-13 cells a side, concatenated (offsets in `small_off`): random and
  small-integer DEMs, a single +-1 bump, 15 % NaN, resolutions (1, 1), (0.5, 1.5) and (30, -30), observers
  anywhere including edges and corners.  `small_raises` marks the cases where the reference raised
  ValueError("node not found") (a NaN in the observer's row east of it); their output is left NaN.
* `large_*`: a few rasters of 200-600 cells a side, among them the reference benchmark's placement
  (linspace(-180, 180, nx) x linspace(-90, 90, nx / 2), observer at x=100, y=50, observer_elev=1).  Their DEMs
  are exact dyadic values from `large_dem` (tests/test_viewshed.py has the same formula; the file keeps a
  checksum).  Only the visibility mask (bit-packed) and the angles of 2048 sampled visible cells are kept.

Usage:  XRS_REFERENCE_ROOT=<reference checkout> python oracle/make_golden_viewshed.py
"""
import inspect
import json
import os
import sys

import numpy as np
import pandas as pd

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_loader  # noqa: E402
from make_golden import encode_default  # noqa: E402

OUT_DIR = os.path.join(os.path.dirname(HERE), "tests", "golden")


class _Values:
    def __init__(self, v):
        self.values = v


class _Raster:
    """What `_viewshed_cpu` reads of a DataArray: shape, values, indexes, sel(method='nearest'), coords, dims."""

    def __init__(self, data, xs, ys):
        self.values = np.array(data)
        self.shape = self.values.shape
        self.dims = ("y", "x")
        self.coords = {"x": xs, "y": ys}
        self.attrs = {}
        self.indexes = {"x": _Values(np.asarray(xs)), "y": _Values(np.asarray(ys))}

    def sel(self, x, y, method):
        assert method == "nearest"
        sx = pd.Index(self.indexes["x"].values).get_indexer(x, method="nearest")
        sy = pd.Index(self.indexes["y"].values).get_indexer(y, method="nearest")
        sel = type("Sel", (), {})()
        sel.x = _Values(self.indexes["x"].values[sx])
        sel.y = _Values(self.indexes["y"].values[sy])
        return sel


def run(data, xs, ys, x, y, observer_elev=0, target_elev=0):
    vs = ref_loader.load("viewshed")
    return np.asarray(vs._viewshed_cpu(_Raster(data, xs, ys), x, y, observer_elev, target_elev).data)


def large_dem(h, w, kind):
    """Exact dyadic test DEMs: a bump plus hashed integer noise ('bump'), small integers ('int')."""
    i = np.arange(h, dtype=np.uint64)[:, None]
    j = np.arange(w, dtype=np.uint64)[None, :]
    noise = (((i * np.uint64(7919) + j * np.uint64(104729)) * np.uint64(2654435761)) % np.uint64(1 << 32)) >> np.uint64(24)
    if kind == "int":
        return (noise % np.uint64(11)).astype(np.float64) - 5.0
    bump = (i * (np.uint64(h - 1) - i)) * (j * (np.uint64(w - 1) - j))
    return bump.astype(np.float64) * (400.0 / float((h - 1) * (h - 1) * (w - 1) * (w - 1))) + noise.astype(np.float64) / 64.0


LARGE = [  # name, h, w, kind, (ew, ns) or None for the benchmark's linspace grid, observer (x, y), obs, tgt, nan
    ("bench", 300, 600, "bump", None, (100.0, 50.0), 1.0, 0.0, 0.0),
    ("int", 400, 400, "int", (1.0, 1.0), (200.0, 117.0), 2.5, 0.0, 0.0),
    ("corner", 256, 512, "bump", (30.0, -30.0), (30.0 * 3, -30.0 * 250), 0.0, 1.5, 0.05),
    ("edge", 500, 200, "bump", (0.5, 1.5), (0.0, 1.5 * 321), 4.0, 0.0, 0.0),
]


def large_case(h, w, kind, res, nan):
    z = large_dem(h, w, kind)
    if res is None:
        xs, ys = np.linspace(-180, 180, w), np.linspace(-90, 90, h)
    else:
        xs, ys = np.arange(w) * res[0], np.arange(h) * res[1]
    if nan:
        i = np.arange(h)[:, None]
        j = np.arange(w)[None, :]
        # NaN cells, none in rows 2 mod 8 (the observer's row: the reference raises on a NaN east of it)
        z = np.where((((i * 31 + j * 17) % 97) < int(nan * 97)) & (i % 8 != 2), np.nan, z)
    return z, xs, ys


def doc_and_tests():
    g = {}
    data = np.array([[0, 0, 1, 0, 0], [1, 3, 0, 0, 0], [10, 2, 5, 2, -1], [11, 1, 2, 9, 0]])
    g["doc_data"] = data
    g["doc_out"] = run(data, np.linspace(1, 5, 5), np.linspace(1, 4, 4), 3, 2)
    cs = np.linspace(-20, 20, 6)
    xs = (cs[:-1] + cs[1:]) / 2          # datashader's pixel centres
    g["tv_coords"] = xs
    params, outs = [], []
    for obs in (-1, 0, 1):
        for elev in (-1, 0, 1):
            for ci, x in enumerate(xs):
                for ri, y in enumerate(xs):
                    a = np.zeros((5, 5), np.int64)
                    a[ri, ci] = elev
                    params.append((obs, elev, ri, ci))
                    outs.append(run(a, xs, xs, x, y, obs))
    g["tv_params"] = np.array(params, np.int64)
    g["tv_out"] = np.array(outs)
    fp, fo = [], []
    for obs in (5, 2):
        for tgt in (0, 1):
            fp.append((obs, tgt))
            fo.append(run(np.full((5, 4), 1.3), np.arange(4) * 0.5, np.arange(5) * 1.5, 0, 0, obs, tgt))
    g["flat_params"] = np.array(fp, np.float64)
    g["flat_out"] = np.array(fo)
    return g


def small_cases(n=320):
    rng = np.random.default_rng(20261017)
    dems, xs_all, ys_all, outs, off, shapes, params, raises = [], [], [], [], [0], [], [], []
    for k in range(n):
        h, w = (int(v) for v in rng.integers(3, 14, 2))
        fam = k % 4
        if fam == 0:
            z = rng.normal(0.0, 2.0, (h, w))
        elif fam == 1:
            z = rng.integers(-2, 3, (h, w)).astype(np.float64)
        elif fam == 2:
            z = np.zeros((h, w))
            z[rng.integers(h), rng.integers(w)] = rng.choice([-1.0, 1.0])
        else:
            z = rng.normal(0.0, 2.0, (h, w))
            z[rng.random((h, w)) < 0.15] = np.nan
        ew, ns = [(1.0, 1.0), (0.5, 1.5), (30.0, -30.0)][k % 3]
        xs, ys = 10.0 + np.arange(w) * ew, -4.0 + np.arange(h) * ns
        r, c = int(rng.integers(h)), int(rng.integers(w))
        if k % 5 == 0:                       # edges and corners
            r, c = [(0, 0), (h - 1, w - 1), (0, w - 1), (h - 1, 0), (0, c)][(k // 5) % 5]
        obs = [-1.0, 0.0, 1.0, 2.5][k % 4 if fam != 3 else (k // 4) % 4]
        tgt = [0.0, 0.0, 1.5][k % 3 if k % 7 else 2]
        try:
            out = run(z, xs, ys, xs[c], ys[r], obs, tgt)
            raised = 0
        except ValueError as e:
            assert "node not found" in str(e), e
            out = np.full((h, w), np.nan)
            raised = 1
        dems.append(z.ravel())
        xs_all.append(xs)
        ys_all.append(ys)
        outs.append(out.ravel())
        off.append(off[-1] + h * w)
        shapes.append((h, w))
        params.append((xs[c], ys[r], obs, tgt))
        raises.append(raised)
    return {"small_dem": np.concatenate(dems), "small_x": np.concatenate(xs_all), "small_y": np.concatenate(ys_all),
            "small_out": np.concatenate(outs), "small_off": np.array(off, np.int64),
            "small_shape": np.array(shapes, np.int64), "small_params": np.array(params),
            "small_raises": np.array(raises, np.int8)}


def large_cases():
    rng = np.random.default_rng(7)
    g = {}
    for name, h, w, kind, res, (x, y), obs, tgt, nan in LARGE:
        z, xs, ys = large_case(h, w, kind, res, nan)
        out = run(z, xs, ys, x, y, obs, tgt)
        vis = out >= 0
        idx = np.flatnonzero(vis)
        pick = np.sort(rng.choice(idx, size=min(2048, idx.size), replace=False))
        g["large_%s_vis" % name] = np.packbits(vis.ravel())
        g["large_%s_idx" % name] = pick.astype(np.int32)
        g["large_%s_ang" % name] = out.ravel()[pick]
        g["large_%s_sum" % name] = np.array([np.nansum(z), np.isnan(z).sum()])
    return g


def signature():
    vs = ref_loader.load("viewshed")
    return {"viewshed": [[k, encode_default(v.default)]
                         for k, v in inspect.signature(inspect.unwrap(vs.viewshed)).parameters.items()]}


def main():
    g = doc_and_tests()
    g.update(small_cases())
    g.update(large_cases())
    np.savez_compressed(os.path.join(OUT_DIR, "viewshed_reference.npz"), **g)
    with open(os.path.join(OUT_DIR, "viewshed_signature.json"), "w") as f:
        json.dump(signature(), f, indent=1, sort_keys=True)
        f.write("\n")
    print(len(g), "arrays in viewshed_reference.npz;", int(g["small_raises"].sum()), "small cases raised")


if __name__ == "__main__":
    main()

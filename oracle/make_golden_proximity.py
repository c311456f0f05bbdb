"""Generate tests/golden/proximity_reference.npz and proximity_signatures.json from the UNMODIFIED reference.

TEST INFRASTRUCTURE (needs a checkout of the reference, like make_golden.py; the existing golden files are not
touched).

* The reference's own tables for proximity / allocation / direction (xrspatial/tests/test_proximity.py): its 4 x 6
  lon / lat raster, every expected array and the QGIS 8 x 6 table, evaluated from the test file's fixtures with
  `ast` (data only, no source is copied).
* The reference's outputs, through `_process` (proximity.py:401-647), for every mode and metric on seeded
  rasters: integer grids, anisotropic, descending and non-uniform coordinates, and lon / lat spanning the
  antimeridian.  The stub DataArray of ref_loader has no `raster[x]`, so a small adapter supplies the 1-D
  coordinates.
* The six public signatures.

Usage:  XRS_REFERENCE_ROOT=<reference checkout> python oracle/make_golden_proximity.py
"""
import ast
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
TEST_FILE = os.path.join(ref_loader.REF_ROOT, "xrspatial", "tests", "test_proximity.py")
MODES = {"proximity": 0, "allocation": 1, "direction": 2}
METRICS = ("EUCLIDEAN", "MANHATTAN", "GREAT_CIRCLE")


class _Coord:
    def __init__(self, data):
        self.data = data


class _Raster:
    """What `_process` reads of a DataArray: data, dims, shape and raster[name].data."""

    def __init__(self, data, xs, ys, x="x", y="y"):
        self.data, self.dims, self.shape = data, (y, x), data.shape
        self._c = {x: _Coord(xs), y: _Coord(ys)}

    def __getitem__(self, k):
        return self._c[k]


def _fixtures():
    tree = ast.parse(open(TEST_FILE).read())
    out = {}
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and (node.name.startswith("result_") or node.name.startswith("qgis_")):
            node.decorator_list = []
            ns = dict(np=np)
            exec(compile(ast.fix_missing_locations(ast.Module(body=[node], type_ignores=[])), TEST_FILE, "exec"), ns)
            out[node.name] = ns[node.name]()
    return out


def tables():
    g = {}
    g["table_data"] = np.asarray([[0., 0., 0., 0., 0., 2.], [0., 0., 1., 0., 0., 0.],
                                  [0., np.inf, 3., 0., 0., 0.], [4., 0., 0., 0., np.nan, 0.]])
    g["table_lon"] = np.linspace(-20, 20, 6)
    g["table_lat"] = np.linspace(20, -20, 4)
    for name, val in _fixtures().items():
        if isinstance(val, tuple):
            param, arr = val
            g["table_%s__param" % name] = np.asarray(param, dtype=np.float64)
            val = arr
        g["table_%s" % name] = np.asarray(val)
    # the QGIS table's raster: the reference conftest's `raster`, with create_test_raster's coordinates
    import make_golden
    q = np.asarray(make_golden.known_answers()["conftest.raster"], dtype=np.float64)
    g["qgis_data"] = q
    h, w = q.shape
    g["qgis_y"] = np.linspace((h - 1) * 0.5, 0, h)
    g["qgis_x"] = np.linspace(0, (w - 1) * 0.5, w)
    return g


def _cases():
    rng = np.random.default_rng(20261017)
    cases = []
    for k, (h, w) in enumerate([(17, 23), (40, 31), (9, 64), (64, 64), (33, 5), (50, 50)]):
        img = (rng.random((h, w)) < [0.02, 0.1, 0.05, 0.01, 0.2, 0.3][k]).astype(np.float32)
        img *= rng.integers(1, 9, (h, w)).astype(np.float32)
        img[0, 0] = 5.0
        cases.append(("int%d" % k, img, np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64)[::-1].copy()))
    img = (rng.random((30, 40)) < 0.05) * rng.standard_normal((30, 40))
    img[3, 3] = np.nan
    cases.append(("aniso", img, np.arange(40) * 30.0, 1000.0 - np.arange(30) * 12.5))
    cases.append(("nonuniform", (rng.random((25, 35)) < 0.06).astype(np.float64) * 3,
                  np.cumsum(rng.uniform(0.5, 2.0, 35)), np.cumsum(rng.uniform(0.5, 2.0, 25))))
    cases.append(("lonlat", (rng.random((24, 36)) < 0.04).astype(np.float64) * 7,
                  np.linspace(-40, 40, 36), np.linspace(60, -60, 24)))
    cases.append(("antimeridian", (rng.random((20, 40)) < 0.03).astype(np.float64) * 2,
                  np.linspace(-179, 179, 40), np.linspace(-50, 50, 20)))
    return cases


def reference_outputs():
    px = ref_loader.load("proximity")
    g = {}
    for name, img, xs, ys in _cases():
        g["case_%s_data" % name], g["case_%s_x" % name], g["case_%s_y" % name] = img, xs, ys
        for metric in METRICS:
            if metric == "GREAT_CIRCLE" and (np.abs(xs).max() > 180 or np.abs(ys).max() > 90):
                continue   # not lon / lat: the reference raises
            for mode, m in MODES.items():
                g["case_%s_%s_%s" % (name, metric, mode)] = px._process(_Raster(img, xs, ys), "x", "y", [], np.inf,
                                                                          metric, m)
    # the scalar distance functions
    pts = np.array([[142.32, 112.54, 23.23, 43.01], [123.2, 178.0, 82.32, 65.09], [-179.5, 179.5, 10.0, -10.0],
                    [0.0, 0.0, 0.0, 0.0], [-20.0, 20.0, 20.0, -20.0]])
    g["scalar_points"] = pts
    g["scalar_values"] = np.array([[px.euclidean_distance(*p), px.manhattan_distance(*p),
                                    px.great_circle_distance(*p)] for p in pts])
    return g


def signatures():
    px = ref_loader.load("proximity")
    names = ["proximity", "allocation", "direction", "euclidean_distance", "manhattan_distance",
             "great_circle_distance"]
    return {n: [[k, encode_default(v.default)] for k, v in inspect.signature(inspect.unwrap(getattr(px, n))).parameters.items()]
            for n in names}


def main():
    g = tables()
    g.update(reference_outputs())
    np.savez_compressed(os.path.join(OUT_DIR, "proximity_reference.npz"), **g)
    with open(os.path.join(OUT_DIR, "proximity_signatures.json"), "w") as f:
        json.dump(signatures(), f, indent=1, sort_keys=True)
        f.write("\n")
    print(len(g), "arrays in proximity_reference.npz")


if __name__ == "__main__":
    main()

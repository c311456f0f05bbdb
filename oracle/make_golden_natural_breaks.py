"""Generate tests/golden/natural_breaks_reference.npz and natural_breaks_signature.json from the UNMODIFIED
reference.

TEST INFRASTRUCTURE (needs a checkout of the reference, like make_golden_classify.py; the existing golden files
are not touched).

* The reference test file's `result_natural_breaks*` fixtures, evaluated with `ast` (data only).
* natural_breaks (classify.py, NumPy path) on the rasters of make_golden_classify.py -- float32 DEMs with NaN,
  +-inf and quantised ties, float64, int16, int32, all-NaN and single-valued rasters -- for k = 1, 2, 5, 10 and
  500 (above the unique count), num_sample None, 1, 8, 1000, 20000 and one larger than the raster, and the
  arguments the reference rejects.  Every call records its output raster, the breaks and new values it passed
  to `_bin`, the text of each warning, or the exception it raised.
* One raster of 3,145,728 cells, so the seeded shuffle runs at scale.  It is not stored: `gen__<case>` names
  the seed and shape the tests rebuild it from (NumPy's PCG64 stream is stable); its calls store the breaks
  and new values, not the output.
* `_run_numpy_jenks_matrices` on a few sorted samples up to 2000 values: `jenks_data__<tag>`,
  `jenks_lcl__<tag>` and `jenks_var__<tag>`.
* The public signature.

Each call is one entry of the JSON manifest `calls`: [case, kwargs, tag].  Its arrays are `out__<tag>`,
`bins__<tag>`, `newv__<tag>`, `warn__<tag>` (the messages) and `err__<tag>` (an exception's class name).

Usage:  XRS_REFERENCE_ROOT=<reference checkout> python oracle/make_golden_natural_breaks.py
"""
import ast
import inspect
import json
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_loader  # noqa: E402
from make_golden import encode_default  # noqa: E402
from make_golden_classify import TEST_FILE, _first_array, cases as classify_cases  # noqa: E402

OUT_DIR = os.path.join(os.path.dirname(HERE), "tests", "golden")
LARGE = {"big_dem_f32": (20261018, 2048, 1536)}


def large_case(seed, h, w):
    """A smooth float32 DEM with NaN and inf cells; the tests rebuild it with this same code."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    dem = (300 * np.sin(x / 97.0) * np.cos(y / 131.0) + 0.25 * x).astype(np.float32)
    dem += rng.normal(0, 2, dem.shape).astype(np.float32)
    dem[rng.random(dem.shape) < 0.01] = np.nan
    dem[5, 7] = np.inf
    return dem


def _fixtures():
    tree = ast.parse(open(TEST_FILE).read())
    out = {}
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name.startswith("result_natural_breaks"):
            node.decorator_list = []
            ns = dict(np=np)
            exec(compile(ast.fix_missing_locations(ast.Module(body=[node], type_ignores=[])), TEST_FILE, "exec"), ns)
            out[node.name] = ns[node.name]()
    return out


def cases():
    c = classify_cases()
    c["ref_elevation"] = np.asarray(_first_array("input_data", "elevation"))
    rng = np.random.default_rng(20261018)
    c["gamma_ties_f32"] = np.round(rng.gamma(2.0, 30.0, (70, 90)) * 4).astype(np.float32) / 4
    c["wide_f64"] = rng.normal(0, 1, (40, 60)) * 10.0 ** rng.integers(-6, 7, (40, 60))
    return c


def calls(fx):
    out = []

    def add(case, tag, **kw):
        out.append([case, kw, tag])

    k, _ = fx["result_natural_breaks"]
    add("ref_elevation", "ref_natural_breaks", k=k)
    k, ns, _ = fx["result_natural_breaks_num_sample"]
    add("ref_elevation", "ref_natural_breaks_num_sample", k=k, num_sample=ns)
    add("ref_elevation", "ref_k30", k=30)   # more classes than unique values
    for case in ["dem_f32", "dem_f32_ties", "dem_f32_lognormal", "f64", "i16", "i32", "all_nan_f32", "single_f32",
                 "few_unique_f32", "gamma_ties_f32", "wide_f64"]:
        for kk in (1, 2, 5, 10, 500):
            add(case, "%s_k%d" % (case, kk), k=kk)
        for ns in (None, 1, 8, 1000, 20000, 10 ** 6):
            add(case, "%s_ns%s" % (case, ns), num_sample=ns)
        add(case, case + "_ns1000_k7", num_sample=1000, k=7)
    for kw, tag in (({"k": 0}, "k0"), ({"k": -1}, "kneg1"), ({"k": -3}, "kneg3"), ({"num_sample": 0}, "ns0"),
                    ({"num_sample": -5}, "nsneg5"), ({"num_sample": 100.0}, "nsfloat"), ({"k": 2.5}, "kfloat")):
        add("dem_f32", "dem_f32_bad_" + tag, **kw)
    add("big_dem_f32", "big_default")
    add("big_dem_f32", "big_ns50000_k7", num_sample=50000, k=7)
    return out


def jenks_samples():
    rng = np.random.default_rng(7)
    return {"normal_n50_k3": (rng.normal(0, 1, 50).astype(np.float32), 3),
            "gamma_ties_n700_k5": ((np.round(rng.gamma(1.5, 10.0, 700)) / 2).astype(np.float32), 5),
            "wide_n2000_k7": ((rng.normal(0, 1, 2000) * 10.0 ** rng.integers(-8, 9, 2000)).astype(np.float32), 7),
            "normal_n1200_k12": (rng.normal(100, 20, 1200).astype(np.float32), 12),
            "i16_n333_k5": (rng.integers(-500, 500, 333).astype(np.int16), 5)}


def run():
    cl = ref_loader.load("classify")
    fx = _fixtures()
    cs = cases()
    g = {"case__" + k: v for k, v in cs.items()}
    for name, (seed, h, w) in LARGE.items():
        cs[name] = large_case(seed, h, w)
        g["gen__" + name] = np.asarray([seed, h, w])
    for name, val in fx.items():
        g["fixture__" + name] = np.asarray(val[-1])
    manifest = calls(fx)
    seen = {}
    orig_bin = cl._bin

    def recording_bin(agg, bins, new_values):
        seen["bins"], seen["newv"] = np.asarray(bins), np.asarray(new_values)
        return orig_bin(agg, bins, new_values)

    cl._bin = recording_bin
    try:
        for case, kw, tag in manifest:
            seen.clear()
            agg = ref_loader._StubDataArray(cs[case].copy(), dims=("y", "x"))
            with warnings.catch_warnings(record=True) as caught:
                warnings.simplefilter("always")
                try:
                    res = cl.natural_breaks(agg, **kw)
                    if case not in LARGE:
                        g["out__" + tag] = np.asarray(res.data)
                except Exception as e:  # noqa: BLE001 - the exception's type is the golden value
                    g["err__" + tag] = np.asarray(type(e).__name__)
            msgs = [str(w.message) for w in caught if w.category is Warning]
            if msgs:
                g["warn__" + tag] = np.asarray(msgs)
            if seen:
                g["bins__" + tag], g["newv__" + tag] = seen["bins"], seen["newv"]
            print(tag, g.get("err__" + tag, ""), flush=True)
    finally:
        cl._bin = orig_bin
    g["calls"] = np.asarray(json.dumps(manifest))
    for tag, (data, k) in jenks_samples().items():
        data = np.sort(data)
        lcl, var = cl._run_numpy_jenks_matrices(data, k)
        g["jenks_data__" + tag], g["jenks_lcl__" + tag], g["jenks_var__" + tag] = data, lcl, var
    return g


def signatures():
    cl = ref_loader.load("classify")
    fn = inspect.unwrap(cl.natural_breaks)
    return {"natural_breaks": [[k, encode_default(v.default)] for k, v in inspect.signature(fn).parameters.items()]}


def main():
    g = run()
    np.savez_compressed(os.path.join(OUT_DIR, "natural_breaks_reference.npz"), **g)
    with open(os.path.join(OUT_DIR, "natural_breaks_signature.json"), "w") as f:
        json.dump(signatures(), f, indent=1, sort_keys=True)
        f.write("\n")
    print(len(g), "arrays in natural_breaks_reference.npz")


if __name__ == "__main__":
    main()

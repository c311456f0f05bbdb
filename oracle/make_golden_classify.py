"""Generate tests/golden/classify_reference.npz and classify_signature.json from the UNMODIFIED reference.

TEST INFRASTRUCTURE (needs a checkout of the reference, like make_golden.py; the existing golden files are not
touched).

* The literal fixtures of the reference's xrspatial/tests/test_classify.py: `input_data`'s elevation, the
  arrays of the heavy-tailed test, the `result_*` fixtures' parameters and expected arrays, evaluated with `ast`
  (data only, no source is copied).
* The reference's public functions (classify.py, NumPy path) on those rasters and on seeded ones: float32 DEMs
  with NaN, +-inf and quantised ties, float64, int16 and int32 rasters, all-NaN and single-valued rasters,
  unsorted and duplicate user bins, `binary` values holding NaN and inf, quantile for k = 1 .. 64,
  maximum_breaks beyond the unique count and box_plot with another hinge.  Every call records its output
  raster, the breaks and new values it passed to `_bin` (captured by wrapping the module's `_bin`), what it
  printed, or the exception it raised.
* The nine public signatures.

Each call is one entry of the JSON manifest `calls`: [case, function, kwargs, tag].  Its arrays are
`out__<tag>`, `bins__<tag>` and `newv__<tag>`; `err__<tag>` holds an exception's class name, `stdout__<tag>` the
printed text.  Rasters are `case__<case>`.

Usage:  XRS_REFERENCE_ROOT=<reference checkout> python oracle/make_golden_classify.py
"""
import ast
import contextlib
import inspect
import io
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_loader  # noqa: E402
from make_golden import encode_default  # noqa: E402

OUT_DIR = os.path.join(os.path.dirname(HERE), "tests", "golden")
TEST_FILE = os.path.join(ref_loader.REF_ROOT, "xrspatial", "tests", "test_classify.py")
NAMES = ["binary", "reclassify", "quantile", "percentiles", "box_plot", "equal_interval", "std_mean",
         "head_tail_breaks", "maximum_breaks"]


def _first_array(fn_name, var):
    """The value first assigned to `var` in the test file's function `fn_name`."""
    tree = ast.parse(open(TEST_FILE).read())
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name == fn_name:
            for st in ast.walk(node):
                if isinstance(st, ast.Assign) and any(getattr(t, "id", None) == var for t in st.targets):
                    return eval(compile(ast.Expression(st.value), TEST_FILE, "eval"), {"np": np})
    raise KeyError((fn_name, var))


def _fixtures():
    tree = ast.parse(open(TEST_FILE).read())
    out = {}
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name.startswith("result_") and "natural" not in node.name:
            node.decorator_list = []
            ns = dict(np=np)
            exec(compile(ast.fix_missing_locations(ast.Module(body=[node], type_ignores=[])), TEST_FILE, "exec"), ns)
            out[node.name] = ns[node.name]()
    return out


def cases():
    c = {"ref_elevation": np.asarray(_first_array("input_data", "elevation")),
         "ref_heavy_tailed": np.asarray(_first_array("test_head_tail_breaks_heavy_tailed", "data")),
         "ref_all_same": np.full((4, 5), 7.0), "ref_all_nan": np.full((4, 5), np.nan)}
    rng = np.random.default_rng(20261017)
    y, x = np.mgrid[0:61, 0:77]
    dem = (200 * np.sin(x / 9.0) * np.cos(y / 13.0) + 3 * x + rng.normal(0, 4, x.shape)).astype(np.float32)
    dem[rng.random(dem.shape) < 0.03] = np.nan
    dem[3, 4], dem[10, 70], dem[40, 2] = np.inf, -np.inf, np.inf
    c["dem_f32"] = dem
    c["dem_f32_ties"] = (np.round(dem / 25.0) * 25.0).astype(np.float32)      # heavy ties
    c["dem_f32_lognormal"] = np.where(np.isfinite(dem), rng.lognormal(3, 1.2, dem.shape), dem).astype(np.float32)
    f64 = rng.normal(1000.0, 250.0, (47, 53))
    f64[rng.random(f64.shape) < 0.05] = np.nan
    c["f64"] = f64
    c["i16"] = rng.integers(-300, 900, (33, 41)).astype(np.int16)
    c["i32"] = (rng.integers(-50, 50, (29, 37)) * 1000).astype(np.int32)
    c["all_nan_f32"] = np.full((8, 9), np.nan, np.float32)
    c["single_f32"] = np.full((6, 7), 3.5, np.float32)
    c["few_unique_f32"] = rng.choice(np.array([-2.0, 0.0, 1.5, 7.25], np.float32), (9, 11))
    return c


def calls(fx):
    out = []

    def add(case, fn, tag, **kw):
        out.append([case, fn, kw, tag])

    b_vals, _ = fx["result_binary"]
    add("ref_elevation", "binary", "ref_binary", values=b_vals)
    rb, rv, _ = fx["result_reclassify"]
    add("ref_elevation", "reclassify", "ref_reclassify", bins=rb, new_values=rv)
    add("ref_elevation", "quantile", "ref_quantile", k=fx["result_quantile"][0])
    add("ref_elevation", "quantile", "ref_quantile_k19", k=19)   # more classes than unique values
    add("ref_elevation", "equal_interval", "ref_equal_interval", k=fx["result_equal_interval"][0])
    add("ref_elevation", "equal_interval", "ref_equal_interval_k1", k=1)
    add("ref_all_nan", "equal_interval", "ref_equal_interval_all_nan", k=3)
    add("ref_elevation", "std_mean", "ref_std_mean")
    add("ref_all_same", "std_mean", "ref_std_mean_all_same")
    add("ref_elevation", "head_tail_breaks", "ref_head_tail")
    add("ref_heavy_tailed", "head_tail_breaks", "ref_head_tail_heavy")
    add("ref_elevation", "percentiles", "ref_percentiles")
    add("ref_elevation", "percentiles", "ref_percentiles_custom", pct=[25, 50, 75])
    add("ref_elevation", "percentiles", "ref_percentiles_single", pct=[50])
    add("ref_elevation", "box_plot", "ref_box_plot")
    add("ref_elevation", "maximum_breaks", "ref_maximum_breaks")
    for case in ["dem_f32", "dem_f32_ties", "dem_f32_lognormal", "f64", "i16", "i32", "all_nan_f32", "single_f32",
                 "few_unique_f32"]:
        add(case, "binary", case + "_binary", values=[-25.0, 0.0, 100.0, 125, np.nan, np.inf])
        add(case, "reclassify", case + "_reclassify", bins=[-100, 0, 50.5, 200, 400], new_values=[1, 2, 3, 4, 5])
        add(case, "reclassify", case + "_reclassify_unsorted", bins=[300, -50, 100, 20, 250, 0],
            new_values=[1.5, 2.5, 3.5, 4.5, 5.5, 6.5])
        add(case, "reclassify", case + "_reclassify_dups", bins=[0, 0, 100, 100, 100, np.inf],
            new_values=[10, 20, 30, 40, 50, 16777217])
        for k in ([4, 5, 10] if case != "dem_f32" else range(1, 65)):
            add(case, "quantile", "%s_quantile_k%d" % (case, k), k=k)
        add(case, "percentiles", case + "_percentiles")
        add(case, "percentiles", case + "_percentiles_custom", pct=[0, 2.5, 33.3, 50, 66.7, 97.5, 100])
        add(case, "box_plot", case + "_box_plot")
        add(case, "box_plot", case + "_box_plot_h07", hinge=0.7)
        add(case, "equal_interval", case + "_equal_interval")
        add(case, "equal_interval", case + "_equal_interval_k7", k=7)
        add(case, "std_mean", case + "_std_mean")
        add(case, "head_tail_breaks", case + "_head_tail")
        for k in (5, 2, 1, 9, 500):   # 500: above the unique count of most cases
            add(case, "maximum_breaks", "%s_maximum_breaks_k%d" % (case, k), k=k)
    return out


def run():
    cl = ref_loader.load("classify")
    fx = _fixtures()
    cs = cases()
    g = {"case__" + k: v for k, v in cs.items()}
    for name, val in fx.items():
        g["fixture__" + name] = np.asarray(val[-1] if isinstance(val, tuple) else val)
    manifest = calls(fx)
    seen = {}
    orig_bin = cl._bin

    def recording_bin(agg, bins, new_values):
        seen["bins"], seen["newv"] = np.asarray(bins), np.asarray(new_values)
        return orig_bin(agg, bins, new_values)

    cl._bin = recording_bin
    try:
        for case, fn, kw, tag in manifest:
            seen.clear()
            agg = ref_loader._StubDataArray(cs[case].copy(), dims=("y", "x"))
            buf = io.StringIO()
            try:
                with contextlib.redirect_stdout(buf):
                    res = getattr(cl, fn)(agg, **kw)
                g["out__" + tag] = np.asarray(res.data)
            except Exception as e:  # noqa: BLE001 - the exception's type is the golden value
                g["err__" + tag] = np.asarray(type(e).__name__)
            if seen:
                g["bins__" + tag], g["newv__" + tag] = seen["bins"], seen["newv"]
            if buf.getvalue():
                g["stdout__" + tag] = np.asarray(buf.getvalue())
    finally:
        cl._bin = orig_bin
    for m in manifest:   # JSON cannot hold NaN / inf literally
        m[2] = {k: [x if isinstance(x, int) else repr(float(x)) for x in v] if isinstance(v, list) else v
                for k, v in m[2].items()}
    g["calls"] = np.asarray(json.dumps(manifest))
    return g


def signatures():
    cl = ref_loader.load("classify")
    return {n: [[k, encode_default(v.default)] for k, v in inspect.signature(inspect.unwrap(getattr(cl, n))).parameters.items()]
            for n in NAMES}


def main():
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        g = run()
    np.savez_compressed(os.path.join(OUT_DIR, "classify_reference.npz"), **g)
    with open(os.path.join(OUT_DIR, "classify_signature.json"), "w") as f:
        json.dump(signatures(), f, indent=1, sort_keys=True)
        f.write("\n")
    print(len(g), "arrays in classify_reference.npz")


if __name__ == "__main__":
    main()

"""Generate tests/golden/local_reference.npz and local_signature.json from the UNMODIFIED reference.

TEST INFRASTRUCTURE (needs a checkout of the reference, like make_golden.py; the existing golden files are not
touched).  Every array comes from the reference's own local.py functions, called on a Dataset stand-in.

* Dataset s: `s{s}_names` (its variables in order), `s{s}_all` (its leading variables of one dtype, stacked) and
  `s{s}_v{j}` (each later variable j).
* call i: row i of `calls` (Dataset index, function, func, ref_var, data_vars joined by commas, "" for None),
  and either `c{i}_out` (the result's values; combine also `c{i}_keyid` and `c{i}_key{j}`, the key tuples' column
  j) or a row of `errors` (i, exception type name, message).
* The JSON holds the nine public signatures and the argument errors of calls that need no data: each with the
  function, the Dataset's variable names (or a non-Dataset stand-in), the arguments, the exception and its message.

Usage:  XRS_REFERENCE_ROOT=<reference checkout> python oracle/make_golden_local.py
"""
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

OUT_DIR = os.path.join(os.path.dirname(HERE), "tests", "golden")
FUNCS = ["cell_stats", "combine", "lesser_frequency", "equal_frequency", "greater_frequency", "lowest_position",
         "highest_position", "popularity", "rank"]
STATS = ["sum", "mean", "median", "min", "max", "std"]
REF_FUNCS = {"lesser_frequency", "equal_frequency", "greater_frequency", "popularity", "rank"}
TYPES = ["float16", "float32", "float64", "int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64",
         "bool"]


class _Var:
    def __init__(self, data):
        self.data = data


class _Dataset(dict):
    """What local.py uses of a Dataset: isinstance, data_vars and ds[name].data."""

    @property
    def data_vars(self):
        return list(self.keys())

    def __getitem__(self, k):
        return _Var(dict.__getitem__(self, k))


def calls_on(names):
    """Every (function, func, ref_var, data_vars) call on a Dataset whose last variable is the ref: the other
    variables are the data."""
    dv = names[:-1]
    out = [("cell_stats", f, None, dv) for f in STATS] + [(f, None, None, dv) for f in
                                                          ("combine", "lowest_position", "highest_position")]
    return out + [(f, None, names[-1], None) for f in sorted(REF_FUNCS)]


def run(loc, call, ds):
    fn, func, ref, dv = call
    f = getattr(loc, fn)
    if fn == "cell_stats":
        return f(ds, dv, func)
    if ref is not None:
        return f(ds, ref, dv)
    return f(ds, dv)


def stack(rng, K, H, W, kind, dtype="float64"):
    if kind == "few":       # small integers: repeats, ties, popularity
        a = rng.integers(-3, 4, (K, H, W)).astype(dtype)
    elif kind == "zeros":   # +-0.0 ties around small values
        a = rng.integers(-1, 2, (K, H, W)).astype(dtype) * rng.choice([0.0, 1.0], (K, H, W))
        a = np.where(rng.random((K, H, W)) < 0.5, -a, a).astype(dtype)
        a[a == 0] = np.where(rng.random((a == 0).sum()) < 0.5, -0.0, 0.0)
    else:                   # spread magnitudes: rounding of sums, means and std
        a = (rng.standard_normal((K, H, W)) * 10.0 ** rng.integers(-4, 5, (K, H, W))).astype(dtype)
    return a


def seeded_cases(rng):
    cases = []
    for K in (1, 2, 3, 7, 8, 9, 16, 17, 128, 129, 200):
        H, W = (6, 7) if K < 100 else (3, 5)
        for kind in ("few", "zeros", "spread"):
            a = stack(rng, K, H, W, kind)
            if kind != "zeros":
                a[0, 0, 1] = np.nan
                a[K - 1, 1, 2] = np.nan
                a[rng.integers(0, K), 2, 3] = np.inf
                a[rng.integers(0, K), 2, 4] = -np.inf
            names = ["v%d" % j for j in range(K)] + ["ref"]
            ref = rng.integers(0, K + 3, (H, W)).astype(np.int64)   # rank / popularity indices, some beyond
            ref[0, 0] = -1
            cases.append((names, list(a) + [ref], calls_on(names)))
    return cases


def typed(rng, dt, shape):
    if dt == "bool":
        return rng.random(shape) < 0.5
    if dt.startswith("float"):
        a = rng.integers(-3, 4, shape).astype(dt)
        m = rng.random(shape) < 0.3
        a[m] = (rng.standard_normal(m.sum()) * 1e3).astype(dt)
        a[(a == 0) & (rng.random(shape) < 0.5)] = -0.0
        return a
    info = np.iinfo(dt)
    hi = min(int(info.max), 2 ** 63 - 1)
    pool = np.array([info.min, info.min + 1, 0, 1, 2, 3, hi - 1, hi], dtype=dt)
    return np.where(rng.random(shape) < 0.5, pool[rng.integers(0, len(pool), shape)],
                    rng.integers(0, 4, shape).astype(dt))


def type_cases(rng):
    """every cell type alone (three layers), then mixed stacks, with refs of every type"""
    cases = []
    H, W = 5, 6
    for dt in TYPES:
        names = ["a", "b", "c", "ref"]
        vs = [typed(rng, dt, (H, W)) for _ in range(3)]
        ref = rng.integers(0, 5, (H, W)).astype(dt if dt != "bool" and not dt.startswith("float") else "int32")
        cases.append((names, vs + [ref], calls_on(names)))
    mixes = [["int64", "float64", "bool"], ["uint8", "int8", "bool"], ["bool", "bool", "int16"],
             ["float32", "uint64", "int32"], ["float16", "int64"], ["uint32", "float32", "bool", "int8"]]
    for m in mixes:
        names = ["m%d" % j for j in range(len(m))] + ["ref"]
        vs = [typed(rng, dt, (H, W)) for dt in m]
        cases.append((names, vs + [rng.integers(-1, len(m) + 2, (H, W)).astype(np.int16)], calls_on(names)))
    # Python's exact int / float comparison against float64 rounding: 2**53 + 1 and 2.0**53
    big = np.array([[2 ** 53 + 1, 2 ** 53, -(2 ** 53) - 1, 5]], np.int64)
    flt = np.array([[2.0 ** 53, 2.0 ** 53 + 2, -(2.0 ** 53), 5.0]])
    for order in ((big, flt), (flt, big)):
        names = ["p", "q", "ref"]
        cases.append((names, list(order) + [np.array([[1, 2, 1, 2]], np.int64)], calls_on(names)))
    for dt in TYPES:   # every ref type against float64 and int64 data
        if dt == "bool":
            refv = np.array([[True, False, True, False]])
        elif dt.startswith("float"):
            refv = np.array([[1.0, np.nan, np.inf, -2.0]], dt)
        else:
            refv = np.array([[1, 0, 2, 3]], dt)
        names = ["d", "e", "ref"]
        d = np.array([[1.0, 0.0, 1e300, -2.0000001]])
        e = np.array([[1, 0, 2 ** 62, -2]], np.int64)
        for fn in ("lesser_frequency", "equal_frequency", "greater_frequency"):
            cases.append((names, [d, e, refv], [(fn, None, "ref", None)]))
    return cases


def rounding_cases():
    """float16 / float32 / int refs against float64 and int data that round onto, past or below them"""
    cases = []
    f16 = [1.0, 2048.0, 65504.0, 0.1, -0.0]
    f32 = [1.0, 16777216.0, 3.4028235e38, 0.1, -0.0]
    for refs, dt in ((f16, "float16"), (f32, "float32"), (f32, "float64")):
        r = np.array(refs, dt)
        with np.errstate(over="ignore"):
            ulp = np.spacing(np.nextafter(r, np.zeros_like(r))).astype(np.float64)   # finite below the largest
        data = []
        for s in (0.0, 0.49, 0.5, 0.51, 1.0, -0.5, -0.51):
            data.append(r.astype(np.float64) + s * ulp)
        data.append(np.where(r == 0, 1e-300, r.astype(np.float64) * 1e300))
        names = ["d%d" % j for j in range(len(data))] + ["i0", "i1", "ref"]
        ints = [np.array([1, 2049, 65505, 0, 0], np.int64), np.array([2, 16777217, 2 ** 60 + 2 ** 36 + 1, 0, -1],
                                                                       np.int64)]
        vs = [v.reshape(1, -1) for v in data] + [v.reshape(1, -1) for v in ints] + [r.reshape(1, -1)]
        for fn in ("lesser_frequency", "equal_frequency", "greater_frequency"):
            cases.append((names, vs, [(fn, None, "ref", None)]))
    for dt in ("int64", "uint64", "int32"):
        names = ["d", "i", "ref"]
        refv = np.array([[2 ** 53 + 1, 2 ** 53, 7, 0]], dt) if dt != "int32" else np.array([[2 ** 31 - 1, 7, 0, 1]], dt)
        d = np.array([[2.0 ** 53, 2.0 ** 53, 7.0000001, -0.0]])
        i = refv.astype(np.int64)
        for fn in ("lesser_frequency", "equal_frequency", "greater_frequency"):
            cases.append((names, [d, i, refv], [(fn, None, "ref", None)]))
    return cases


def index_cases(rng):
    """rank / popularity indices: 0, negative, beyond K, wrapping uint8 / int8, bool refs, and the errors"""
    cases = []
    H, W = 4, 5
    base = rng.integers(0, 3, (4, H, W)).astype(np.float64)
    base[:, 0, 0] = [1.0, 1.0, 1.0, 1.0]       # one distinct value
    base[:, 0, 1] = [3.0, 1.0, 2.0, 0.0]       # all distinct
    base[:, 0, 2] = [0.0, -0.0, 1.0, -0.0]     # +-0.0 as one value
    base[:, 0, 3] = [-0.0, 0.0, -0.0, 0.0]
    names = ["a", "b", "c", "d", "ref"]
    for dt, vals in (("uint8", [0, 1, 2, 3, 4, 5, 255]), ("int8", [-128, -1, 0, 1, 2, 3, 127]),
                     ("int64", [-1, 0, 1, 2, 3, 5, 2 ** 62]), ("uint64", [0, 1, 2, 3, 4, 2 ** 63 - 1, 9]),
                     ("bool", [True, False]), ("int16", [-2, -1, 0, 1, 2, 3, 4])):
        ref = np.array(vals, dt)[rng.integers(0, len(vals), (H, W))]
        for fn in ("rank", "popularity"):
            cases.append((names, list(base) + [ref], [(fn, None, "ref", None)]))
    # errors: an index below -length, a float ref reaching the index; and a float ref that never does
    for fn, ref, data in (("rank", -5, base), ("rank", -3, base), ("popularity", -3, base),
                          ("rank", 2.0, base), ("popularity", 2.0, base),
                          ("rank", 9.0, base), ("popularity", 1.5, base[:, :1, :2])):
        dt = np.float32 if isinstance(ref, float) else np.int64
        r = np.full(data.shape[1:], ref, dt)
        cases.append((names, list(data) + [r], [(fn, None, "ref", None)]))
    nanref = np.full((H, W), np.nan, np.float32)
    for fn in ("lesser_frequency", "equal_frequency", "greater_frequency", "rank"):
        cases.append((names, list(base[:, :1, :1]) + [nanref[:1, :1]],
                      [(fn, None, "ref", None)]))
    return cases


def combine_cases(rng):
    cases = []
    for H, W, K, n in ((20, 30, 3, 2), (16, 16, 2, 1000), (12, 10, 5, 3)):
        a = rng.integers(0, n, (K, H, W)).astype(np.float64)
        a[0, 1, 1] = np.nan
        a[a == 0] = np.where(rng.random((a == 0).sum()) < 0.5, -0.0, 0.0)
        names = ["v%d" % j for j in range(K)]
        cases.append((names, list(a), [("combine", None, None, None)]))
    names = ["i", "f", "b"]
    vs = [rng.integers(0, 3, (10, 12)).astype(np.uint16), rng.integers(0, 2, (10, 12)).astype(np.float32),
          rng.random((10, 12)) < 0.5]
    cases.append((names, vs, [("combine", None, None, None)]))
    return cases


def fixture_cases():
    arr = np.full((4, 4), 2)
    arr1 = np.array([[np.nan, 4, 2, 0], [2, 3, np.nan, 1], [5, 1, 2, 0], [1, 3, 2, np.nan]])
    arr2 = np.array([[3, 1, 1, 2], [4, 1, 2, 5], [0, 0, 0, 0], [np.nan, 1, 1, 1]])
    arr3 = np.array([[3, 3, 2, 0], [4, 1, 3, 1], [6, 1, 2, 2], [0, 0, 1, 1]])
    names = ["arr", "arr1", "arr2", "arr3"]
    vs = [arr, arr1, arr2, arr3]
    cases = [(names[1:], vs[1:], [("cell_stats", f, None, None) for f in STATS] + [
        (f, None, None, None) for f in ("combine", "lowest_position", "highest_position")] + [
        ("cell_stats", "sum", None, ["arr1", "arr3"])])]
    for fn in sorted(REF_FUNCS):
        cases.append((names, vs, [(fn, None, "arr", None), (fn, None, "arr", ["arr1", "arr2"])]))
    return cases


def argument_errors(loc):
    """(function, variable names or a stand-in name, args, kwargs) for every argument check, in order"""
    names = ["a", "b", "c"]
    calls = []
    for fn in FUNCS:
        has_ref = fn in REF_FUNCS
        extra = {"ref_var": "c"} if has_ref else {}
        calls.append((fn, "ndarray", dict(extra)))
        calls.append((fn, "dict", dict(extra)))
        if fn == "cell_stats":
            calls.append((fn, names, {"func": "mode"}))
            calls.append((fn, "ndarray", {"func": "mode"}))
        if has_ref:
            calls.append((fn, names, {"ref_var": 3}))
            calls.append((fn, names, {"ref_var": "z"}))
            calls.append((fn, names, {"ref_var": "z", "data_vars": "a"}))
            calls.append((fn, names, {"ref_var": "c", "data_vars": ["a", "c"]}))
        calls.append((fn, names, dict(extra, data_vars="a")))
        calls.append((fn, names, dict(extra, data_vars=["a", 1])))
        calls.append((fn, names, dict(extra, data_vars=["a", "q"])))
    out = []
    for fn, raster, kw in calls:
        if isinstance(raster, list):
            ds = _Dataset({k: np.zeros((2, 3)) for k in raster})
        else:
            ds = np.zeros((2, 3)) if raster == "ndarray" else {"a": 1}
        try:
            getattr(loc, fn)(ds, **kw)
        except Exception as e:   # noqa: BLE001 - the reference's exception is the datum
            out.append([fn, raster, kw, type(e).__name__, str(e)])
            continue
        raise AssertionError("no error: %s %s %s" % (fn, raster, kw))
    return out


def main():
    loc = ref_loader.load("local")
    sys.modules["xarray"].Dataset = _Dataset   # local.py looks xr.Dataset up at call time
    rng = np.random.default_rng(20261019)
    cases = fixture_cases() + seeded_cases(rng) + type_cases(rng) + rounding_cases() + index_cases(rng) + \
        combine_cases(rng)
    out, rows, errors = {}, [], []
    i = 0
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")   # the reference's scalar overflow in `ref - 1`, inf - inf
        for c, (names, vs, calls) in enumerate(cases):
            ds = _Dataset(zip(names, vs))
            out["s%d_names" % c] = np.array(names)
            n = 1
            while n < len(vs) and vs[n].dtype == vs[0].dtype and vs[n].shape == vs[0].shape:
                n += 1
            out["s%d_all" % c] = np.stack(vs[:n])
            for j in range(n, len(vs)):
                out["s%d_v%d" % (c, j)] = vs[j]
            for call in calls:
                p = "c%d_" % i
                rows.append([str(c), call[0], call[1] or "", call[2] or "", ",".join(call[3] or [])])
                i += 1
                try:
                    r = run(loc, call, ds)
                except (IndexError, TypeError) as e:
                    errors.append([str(i - 1), type(e).__name__, str(e)])
                    continue
                out[p + "out"] = np.asarray(r.data)
                if call[0] == "combine":
                    key = r.attrs["key"]
                    out[p + "keyid"] = np.array(list(key.keys()), np.int64)
                    tuples = list(key.values())
                    for j in range(len(tuples[0]) if tuples else 0):
                        out[p + "key%d" % j] = np.array([t[j] for t in tuples])
    out["calls"] = np.array(rows)
    out["errors"] = np.array(errors)
    np.savez_compressed(os.path.join(OUT_DIR, "local_reference.npz"), **out)

    def params(f):
        return [[k, encode_default(v.default)] for k, v in inspect.signature(inspect.unwrap(f)).parameters.items()]
    sig = {"signatures": {f: params(getattr(loc, f)) for f in FUNCS}, "errors": argument_errors(loc)}
    with open(os.path.join(OUT_DIR, "local_signature.json"), "w") as f:
        json.dump(sig, f, indent=1)
    print("%d calls" % i)


if __name__ == "__main__":
    main()

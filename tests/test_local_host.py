"""local without a GPU: local_rule.cuh compiled with g++ and run cell by cell through the package's own argument
checks, cell-type table and result typing, against every golden array of the unmodified reference (bit for bit,
dtype and NaN pattern included); the public signatures; and the argument errors raised before any device work."""
import ctypes
import inspect
import json
import os
import subprocess

import numpy as np
import pytest
import torch

import xrspatial_b200 as xb
from xrspatial_b200 import _lib, local

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "xarray-spatial_b200", "csrc", "local_rule.cuh")
GOLDEN = os.path.join(ROOT, "tests", "golden")
REF_FUNCS = {"lesser_frequency", "equal_frequency", "greater_frequency", "popularity", "rank"}


def golden():
    return dict(np.load(os.path.join(GOLDEN, "local_reference.npz"), allow_pickle=False))


def golden_signature():
    with open(os.path.join(GOLDEN, "local_signature.json")) as f:
        return json.load(f)


def golden_cases(g):
    """(index, dict of the Dataset's variables, function, func, ref_var, data_vars, expected) per golden call;
    expected is ("out", array, key) or ("err", type name, message)."""
    errors = {int(i): (t, m) for i, t, m in g["errors"]}
    datasets = {}
    for i, (c, fn, func, ref, dv) in enumerate(g["calls"]):
        if c not in datasets:
            names = list(g["s%s_names" % c])
            vs = list(g["s%s_all" % c])
            vs += [g["s%s_v%d" % (c, j)] for j in range(len(vs), len(names))]
            datasets[c] = dict(zip(names, vs))
        if i in errors:
            want = ("err",) + errors[i]
        else:
            key = None
            if fn == "combine":
                ids = g["c%d_keyid" % i]
                cols = [g["c%d_key%d" % (i, j)].tolist() for j in range(len(datasets[c]) if len(ids) else 0)
                        if "c%d_key%d" % (i, j) in g]
                key = dict(zip(ids.tolist(), zip(*cols)))
            want = ("out", g["c%d_out" % i], key)
        yield i, datasets[c], fn, func or None, ref or None, (dv.split(",") if dv else None), want


_HOST_SRC = r"""
#include <unordered_map>
#include <vector>
using namespace xrs::lc;
static Val read(const int64_t *l, int64_t r, int64_t c) {
    const char *row = (const char *)l[0] + r * l[1];
    switch (l[2]) {
        case XRS_F32: return load(((const float *)row)[c]);
        case XRS_F64: return load(((const double *)row)[c]);
        case XRS_I32: return load(((const int32_t *)row)[c]);
        case XRS_I64: case XRS_U64: return load(((const int64_t *)row)[c]);
        case XRS_I16: return load(((const int16_t *)row)[c]);
        case XRS_U16: return load(((const uint16_t *)row)[c]);
        case XRS_I8: return load(((const int8_t *)row)[c]);
        case XRS_U8: return load(((const uint8_t *)row)[c]);
        case XRS_U32: return load(((const uint32_t *)row)[c]);
        default: return ival(((const uint8_t *)row)[c] != 0, kBool);
    }
}
extern "C" unsigned lc_cells(const int64_t *layers, int64_t K, int64_t H, int64_t W, int op, int ak,
                             const int64_t *ref, int ref_f16, int64_t *out, uint8_t *kinds) {
    unsigned flags = 0;
    for (int64_t k = 0; k < H * W; ++k) {
        const int64_t r = k / W, c = k % W;
        auto x = [&](int64_t j) { return read(layers + 3 * j, r, c); };
        Ref rf{};
        if (ref) rf = make_ref(read(ref, r, c), (int)ref[2], ref_f16 != 0);
        const Result res = cell(op, K, ak, x, rf);
        out[k] = res.bits;
        kinds[k] = (uint8_t)res.kind;
        flags |= res.flags;
    }
    return flags;
}
// combine in row-major order: ids[k] (-1 for NaN), reps[id - 1] = the id's first cell; returns the flags
extern "C" unsigned lc_combine(const int64_t *layers, int64_t K, int64_t H, int64_t W, int64_t *ids, int64_t *reps) {
    std::unordered_multimap<uint64_t, int64_t> seen;
    int64_t n = 0;
    unsigned flags = 0;
    for (int64_t k = 0; k < H * W; ++k) {
        auto x = [&](int64_t j) { return read(layers + 3 * j, k / W, k % W); };
        bool nan = false;
        for (int64_t j = 0; j < K; ++j) nan |= is_nan(x(j));
        ids[k] = -1;
        if (nan) { flags |= kFlagNan; continue; }
        const uint64_t h = tuple_hash(K, x);
        auto range = seen.equal_range(h);
        for (auto it = range.first; it != range.second; ++it) {
            const int64_t u = it->second;
            auto y = [&](int64_t j) { return read(layers + 3 * j, reps[u] / W, reps[u] % W); };
            if (tuple_equal(K, x, y)) { ids[k] = u + 1; break; }
        }
        if (ids[k] < 0) { reps[n] = k; seen.emplace(h, n); ids[k] = ++n; }
    }
    return flags;
}
"""


def build_host(directory):
    cpp, so = os.path.join(directory, "lc.cpp"), os.path.join(directory, "lc.so")
    with open(cpp, "w") as f:
        f.write('#include "%s"\n' % HEADER + _HOST_SRC)
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, cpp])
    lib = ctypes.CDLL(so)
    P, I64, I = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
    lib.lc_cells.argtypes = [P, I64, I64, I64, I, I, P, I, P, P]
    lib.lc_cells.restype = ctypes.c_uint
    lib.lc_combine.argtypes = [P, I64, I64, I64, P, P]
    lib.lc_combine.restype = ctypes.c_uint
    return lib


def _rows(tensors, codes):
    return (ctypes.c_int64 * (3 * len(tensors)))(*[v for t, c in zip(tensors, codes)
                                                   for v in (t.data_ptr(), t.stride(0) * t.element_size(), c)])


def host_call(lib, fn, raster, func=None, ref_var=None, data_vars=None):
    """The public function's path with the host build of the rule in place of the device."""
    data_vars = local._check(raster, data_vars, ref_var, fn in REF_FUNCS, func if fn == "cell_stats" else None)
    s = local._Stack(raster, data_vars, ref_var, device=False)
    H, W = s.H, s.W
    bits = torch.empty((H, W), dtype=torch.int64)
    if fn == "combine":
        reps = torch.empty(H * W, dtype=torch.int64)
        flags = lib.lc_combine(_rows(s.tensors, s.codes), s.K, H, W, bits.data_ptr(), reps.data_ptr())
        u = int(bits.max()) if H * W else 0
        reps = reps[:max(u, 0)]
        cols = [local._gather(t, c, reps // W, reps % W) for t, c in zip(s.tensors, s.codes)]
        out = local._finish("combine", s.ak, bits, None, flags)
        return s.container(out), {i + 1: t for i, t in enumerate(zip(*cols))}
    op = local.funcs[func] if fn == "cell_stats" else local.OPS[fn]
    kinds = torch.empty((H, W), dtype=torch.uint8)
    ref = _rows(s.tensors[s.K:], s.codes[s.K:]) if ref_var is not None else None
    flags = lib.lc_cells(_rows(s.tensors[:s.K], s.codes), s.K, H, W, op, s.ak, ref,
                         int(ref_var is not None and s.f16[s.K]), bits.data_ptr(), kinds.data_ptr())
    out = local._finish(op, s.ak, bits, kinds, flags, local._ref_type(s) if ref_var is not None else None)
    return s.container(out), None


def same_result(got, want):
    """Equal dtype, shape and values, the sign of zero and the NaN pattern included (NaN payloads may differ)."""
    got = np.asarray(got)
    if got.dtype != want.dtype or got.shape != want.shape:
        return False
    if want.dtype.kind != "f":
        return np.array_equal(got, want)
    gn, wn = np.isnan(got), np.isnan(want)
    return np.array_equal(gn, wn) and np.array_equal(got[~gn].view(np.int64), want[~wn].view(np.int64))


def same_key(got, want):
    if got.keys() != want.keys():
        return False
    for k in want:
        if len(got[k]) != len(want[k]):
            return False
        for a, b in zip(got[k], want[k]):
            if type(a) is not type(b) or np.float64(a).tobytes() != np.float64(b).tobytes():
                return False
    return True


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    return build_host(str(tmp_path_factory.mktemp("lc")))


def run_golden_case(call, ds_vars, fn, func, ref, dv, want):
    raster = xb.Dataset(ds_vars)
    if want[0] == "err":
        with pytest.raises(Exception) as e:
            call(fn, raster, func, ref, dv)
        assert (type(e.value).__name__, str(e.value)) == want[1:]
        return
    out, key = call(fn, raster, func, ref, dv)
    assert same_result(out, want[1]), (fn, func, out, want[1])
    if fn == "combine":
        assert same_key(key, want[2])


def test_host_rule_reproduces_every_golden_call(host):
    n = 0
    for i, ds_vars, fn, func, ref, dv, want in golden_cases(golden()):
        try:
            run_golden_case(lambda *a: host_call(host, *a), ds_vars, fn, func, ref, dv, want)
        except AssertionError as e:
            raise AssertionError("golden call %d (%s %s): %s" % (i, fn, func, e)) from None
        n += 1
    assert n > 800


def test_golden_covers_every_cell_type_function_and_stack_depth():
    g = golden()
    seen_types, seen_k, seen_fn = set(), set(), set()
    for _, ds_vars, fn, func, ref, dv, _ in golden_cases(g):
        seen_types |= {v.dtype.name for v in ds_vars.values()}
        seen_fn.add(func or fn)
        seen_k.add(len(dv) if dv else len(ds_vars) - (ref is not None))
    assert seen_types >= {"float16", "float32", "float64", "int8", "int16", "int32", "int64", "uint8", "uint16",
                          "uint32", "uint64", "bool"}
    assert seen_k >= {2, 3, 7, 8, 9, 16, 17, 128, 129, 200}
    assert seen_fn >= {"sum", "mean", "median", "min", "max", "std", "combine"} | REF_FUNCS | {
        "lowest_position", "highest_position"}


@pytest.mark.parametrize("K", [1, 2, 7, 8, 9, 15, 16, 17, 64, 127, 128, 129, 130, 300, 1000, 1030])
def test_host_sum_std_and_extremes_match_numpy_at_every_depth(host, K):
    """np.sum / np.std / np.mean bit for bit, and np.max / np.min by value, over float64 stacks beyond the golden
    depths"""
    rng = np.random.default_rng(K)
    a = rng.standard_normal((K, 3, 4)) * 10.0 ** rng.integers(-3, 4, (K, 3, 4))
    a[:, 0, :] = np.where(rng.random((K, 4)) < 0.5, -0.0, 0.0)
    names = ["v%d" % j for j in range(K)]
    raster = xb.Dataset(dict(zip(names, a)))
    for func, np_func in (("sum", np.sum), ("std", np.std), ("max", np.max), ("min", np.min), ("mean", np.mean)):
        if K == 1:
            with pytest.raises(TypeError, match="0-d"):
                host_call(host, "cell_stats", raster, func, data_vars=names)
            continue
        got, _ = host_call(host, "cell_stats", raster, func)
        want = np.array([np_func(tuple(a[:, r, c].tolist())) for r in range(3) for c in range(4)]).reshape(3, 4)
        if func in ("max", "min"):
            # which of equal +-0.0 np.max / np.min return depends on the SIMD width NumPy dispatches on this CPU;
            # the goldens pin it, so only values are compared here (row 0 holds only +-0.0)
            assert np.array_equal(got, want), func
            continue
        assert same_result(got, want), func


@pytest.mark.parametrize("d", [1.0, 1.0 + 2 ** -11, 1.0 + 3 * 2 ** -11, 65504.0, 65519.99, 65520.0, 6.1e-5,
                               2.0 ** -24, 2.0 ** -25, 3 * 2.0 ** -25, 1e-30, 0.1, 2049.0, 2051.0, -2051.0])
def test_host_float16_rounding_matches_numpy(host, d):
    """equal_frequency against a float16 ref: the data value rounds to float16 exactly as NumPy rounds it"""
    ref = np.array([[np.float16(d)]], np.float16)
    raster = xb.Dataset({"a": np.array([[d]]), "b": np.array([[d]]), "ref": ref})
    got, _ = host_call(host, "equal_frequency", raster, ref_var="ref")
    assert int(got[0, 0]) == 2 * int(ref[0, 0] == d)


def test_signatures_match_the_reference():
    from make_golden import encode_default
    sig = golden_signature()["signatures"]
    assert len(sig) == 9
    for name, params in sig.items():
        f = getattr(xb.local, name)
        got = [[k, encode_default(v.default)] for k, v in inspect.signature(f).parameters.items()]
        assert got == params, name


def test_argument_errors_match_the_reference_without_a_device():
    errors = golden_signature()["errors"]
    assert len(errors) > 60
    for fn, raster, kw, etype, message in errors:
        if isinstance(raster, list):
            ds = xb.Dataset({k: np.zeros((2, 3)) for k in raster})
        else:
            ds = np.zeros((2, 3)) if raster == "ndarray" else {"a": 1}
        with pytest.raises(Exception) as e:
            getattr(xb.local, fn)(ds, **kw)
        assert (type(e.value).__name__, str(e.value)) == (etype, message), (fn, raster, kw)


def test_deviations_raise_before_any_device_work():
    with pytest.raises(ValueError, match="same 2-D shape"):
        xb.local.cell_stats(xb.Dataset({"a": xb.DataArray(np.zeros((2, 3)), dims=("y", "x")),
                                        "b": xb.DataArray(np.zeros((3, 2)), dims=("v", "u"))}))
    with pytest.raises(ValueError, match="2-D"):
        xb.local.cell_stats(xb.Dataset({"a": np.zeros((2, 3, 2)), "b": np.zeros((2, 3, 2))}))
    with pytest.raises(ValueError, match="above 2\\*\\*63"):
        xb.local.combine(xb.Dataset({"a": np.array([[2 ** 63]], np.uint64), "b": np.zeros((1, 1))}))


def test_c_entry_points_check_arguments_before_any_cuda_call():
    lib = _lib.lib()
    buf = (ctypes.c_double * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    F32 = _lib.ZONAL_CELLS["float32"]
    layers = (ctypes.c_int64 * 6)(ctypes.addressof(buf), 16, F32, ctypes.addressof(buf), 16, F32)
    bad_code = (ctypes.c_int64 * 6)(ctypes.addressof(buf), 16, F32, ctypes.addressof(buf), 16, 11)
    bad_pitch = (ctypes.c_int64 * 6)(ctypes.addressof(buf), 8, F32, ctypes.addressof(buf), 16, F32)
    need = ctypes.c_int64()
    assert lib.xrs_local_combine_scratch_bytes(100, 100, ctypes.byref(need)) == _lib.XRS_OK
    assert need.value == 8 * 32768
    cases = [
        (lambda: lib.xrs_local_cells(layers, 2, p, 4, 4, 13, 0, None, 0, 0, 0, p, 32, p, 4, p, None), b"op"),
        (lambda: lib.xrs_local_cells(layers, 2, p, 4, 4, 0, 3, None, 0, 0, 0, p, 32, p, 4, p, None), b"kind"),
        (lambda: lib.xrs_local_cells(layers, 2, p, 4, 4, 0, 0, None, 0, 0, 0, p, 16, p, 4, p, None), b"output pitch"),
        (lambda: lib.xrs_local_cells(bad_code, 2, p, 4, 4, 0, 0, None, 0, 0, 0, p, 32, p, 4, p, None), b"cell type"),
        (lambda: lib.xrs_local_cells(bad_pitch, 2, p, 4, 4, 0, 0, None, 0, 0, 0, p, 32, p, 4, p, None),
         b"input pitch"),
        (lambda: lib.xrs_local_cells(layers, 2, p, 4, 4, 6, 0, None, 16, F32, 0, p, 32, p, 4, p, None), b"NULL"),
        (lambda: lib.xrs_local_cells(layers, 2, p, 4, 4, 6, 0, p, 32, 1, 1, p, 32, p, 4, p, None), b"float16"),
        (lambda: lib.xrs_local_cells(layers, 2, p, 4, 4, 12, 0, p, 16, F32, 0, p, 32, None, 4, p, None), b"kinds"),
        (lambda: lib.xrs_local_cells(layers, 0, p, 4, 4, 0, 0, None, 0, 0, 0, p, 32, p, 4, p, None), b"no layers"),
        (lambda: lib.xrs_local_combine(layers, 2, p, 4, 4, 0, p, 8, None, p, 32, p, None), b"too small"),
        (lambda: lib.xrs_local_combine(layers, 2, p, 4, 4, 2, p, 1 << 10, None, p, 32, p, None), b"phase"),
        (lambda: lib.xrs_local_combine(layers, 2, p, 4, 4, 1, p, 1 << 10, None, p, 32, p, None), b"reps"),
    ]
    for call, words in cases:
        assert call() == _lib.XRS_EINVAL, words
        assert words in lib.xrs_last_error_string(), (words, lib.xrs_last_error_string())

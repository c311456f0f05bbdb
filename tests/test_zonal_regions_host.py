"""zonal regions / trim / crop without a GPU: zonal_regions_rule.cuh compiled with g++ and labelled by a host
union-find against every golden `regions` array of the unmodified reference, the public signatures, the canvas
arithmetic, and the argument errors raised before any device work."""
import ctypes
import inspect
import json
import os
import subprocess

import numpy as np
import pytest

import xrspatial_b200 as xb
from xrspatial_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "xarray-spatial_b200", "csrc", "zonal_regions_rule.cuh")
GOLDEN = os.path.join(ROOT, "tests", "golden")
SUFFIX = {"float32": "f32", "float64": "f64", "int8": "i8", "int16": "i16", "int32": "i32", "int64": "i64",
          "uint8": "u8", "uint16": "u16", "uint32": "u32", "uint64": "u64"}


def golden():
    return dict(np.load(os.path.join(GOLDEN, "zonal_regions_reference.npz"), allow_pickle=False))


def golden_signature():
    with open(os.path.join(GOLDEN, "zonal_regions_signature.json")) as f:
        return json.load(f)


def region_cases(g):
    i = 0
    while "reg%d_in" % i in g:
        yield i, g["reg%d_in" % i], int(g["reg_n"][i]), g["reg%d_out" % i]
        i += 1


def bounds_cases(g):
    i = 0
    while "bnd%d_in" % i in g:
        v = g["bnd%d_values" % i]
        vals = tuple(int(x) for x in v) if v.dtype.kind == "i" else tuple(float(x) for x in v)
        yield i, g["bnd%d_in" % i], vals, int(g["bnd%d_mode" % i]), tuple(int(x) for x in g["bnd%d_out" % i])
        i += 1


_HOST_SRC = r"""
#include <vector>
using namespace xrs::zr;
static int64_t find(std::vector<int64_t> &p, int64_t x) {
    while (p[x] != x) x = p[x] = p[p[x]];
    return x;
}
// the rule's codes and edges, unioned one at a time; labels as int64, nan[k] = 1 for NaN cells
template <typename T> static void run(const T *z, int64_t H, int64_t W, int n, int64_t *lab, uint8_t *nan) {
    const int64_t N = H * W;
    std::vector<uint32_t> code(N);
    std::vector<int64_t> p(N), uid(N);
    auto get = [&](int64_t r, int64_t c) { return z[r * W + c]; };
    int64_t u = 0;
    for (int64_t k = 0; k < N; ++k) {
        code[k] = cell_code<T>(n, H, W, k / W, k % W, get);
        p[k] = k;
        if (code[k] & kNew) ++u;
        uid[k] = u;
    }
    for (int64_t k = 0; k < N; ++k)
        for_each_edge(n, H, W, k / W, k % W, code[k], [&](int64_t a, int64_t b) {
            a = find(p, a);
            b = find(p, b);
            if (a < b) p[b] = a;
            else if (b < a) p[a] = b;
        });
    for (int64_t k = 0; k < N; ++k) {
        nan[k] = (code[k] & kNan) != 0;
        lab[k] = nan[k] ? 0 : uid[find(p, k)];
    }
}
#define E(s, T) \
    extern "C" void zr_##s(const T *z, int64_t H, int64_t W, int n, int64_t *lab, uint8_t *nan) { run<T>(z, H, W, n, lab, nan); }
E(f32, float) E(f64, double) E(i8, int8_t) E(i16, int16_t) E(i32, int32_t) E(i64, int64_t) E(u8, uint8_t)
E(u16, uint16_t) E(u32, uint32_t) E(u64, uint64_t)
"""


def build_host(directory):
    """The header's rule plus a host union-find, as a function (array, n) -> labels in the array's cell type."""
    cpp, so = os.path.join(directory, "zr.cpp"), os.path.join(directory, "zr.so")
    with open(cpp, "w") as f:
        f.write('#include "%s"\n' % HEADER + _HOST_SRC)
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, cpp])
    lib = ctypes.CDLL(so)
    P, I64 = ctypes.c_void_p, ctypes.c_int64
    for s in SUFFIX.values():
        getattr(lib, "zr_" + s).argtypes = [P, I64, I64, ctypes.c_int, P, P]

    def labels(a, n):
        a = np.ascontiguousarray(a)
        H, W = a.shape
        lab = np.zeros((H, W), np.int64)
        nan = np.zeros((H, W), np.uint8)
        getattr(lib, "zr_" + SUFFIX[a.dtype.name])(a.ctypes.data, H, W, n, lab.ctypes.data, nan.ctypes.data)
        out = lab.astype(a.dtype)
        if a.dtype.kind == "f":
            out[nan.astype(bool)] = np.nan
        return out
    return labels


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    return build_host(str(tmp_path_factory.mktemp("zr")))


def test_host_rule_reproduces_every_golden_regions_array(host):
    g = golden()
    n_cases = 0
    for i, a, n, ref in region_cases(g):
        got = host(a, n)
        assert got.dtype == ref.dtype
        assert np.array_equal(got, ref, equal_nan=a.dtype.kind == "f"), i
        n_cases += 1
    assert n_cases > 300


def test_golden_covers_every_cell_type_and_both_neighbourhoods():
    g = golden()
    seen = {(a.dtype.name, n) for _, a, n, _ in region_cases(g)}
    for t in SUFFIX:
        assert (t, 4) in seen and (t, 8) in seen, t


@pytest.mark.parametrize("a, n, want", [
    (np.array([[-128, -128]], np.int8), 4, [[1, 2]]),                      # |int8 -128| is -128: no match
    (np.array([[100000, 100001]], np.uint32), 4, [[1, 1]]),              # 100001 - 100000 = 1 is close,
    (np.array([[100001, 100000]], np.uint32), 4, [[1, 1]]),              # 100000 - 100001 wraps, one side joins
    (np.array([[np.inf, np.inf]], np.float64), 4, [[1, 2]]),             # inf - inf is NaN
    (np.array([[1.0, np.inf]], np.float64), 4, [[1, 1]]),                # any finite value matches an inf centre
])
def test_host_rule_on_the_arithmetic_edges(host, a, n, want):
    assert np.array_equal(host(a, n), np.array(want, a.dtype))


def test_signatures_match_the_reference():
    from make_golden import encode_default
    sig = golden_signature()["signatures"]
    for name, params in sig.items():
        f = getattr(xb.zonal, name)
        got = [[k, encode_default(v.default)] for k, v in inspect.signature(f).parameters.items()]
        assert got == params, name
    for name in ("regions", "trim", "crop", "suggest_zonal_canvas"):
        assert getattr(xb, name) is getattr(xb.zonal, name)


def test_canvas_and_full_extent_match_the_reference():
    sig = golden_signature()
    for args, want in sig["canvas"]:
        assert list(xb.suggest_zonal_canvas(*args)) == want, args
    for crs, want in sig["full_extent"].items():
        assert [list(v) for v in xb.zonal.get_full_extent(crs)] == want
    with pytest.raises(KeyError):
        xb.zonal.get_full_extent("Robinson")


def test_argument_errors_without_a_device():
    a = xb.DataArray(np.zeros((4, 4), np.float32), dims=("y", "x"))
    for n in (0, 6, 9):
        with pytest.raises(ValueError, match="neighborhood"):
            xb.regions(a, neighborhood=n)
    h = xb.DataArray(np.zeros((4, 4), np.float16), dims=("y", "x"))
    with pytest.raises(NotImplementedError):
        xb.regions(h)
    with pytest.raises(NotImplementedError):
        xb.trim(h)


def test_c_entry_points_check_arguments_before_any_cuda_call():
    lib = _lib.lib()
    buf = (ctypes.c_double * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    need = ctypes.c_int64()
    F32 = _lib.ZONAL_CELLS["float32"]
    assert lib.xrs_zonal_regions_scratch_bytes(100, 100, ctypes.byref(need)) == _lib.XRS_OK
    assert need.value >= 10 * 100 * 100
    assert lib.xrs_zonal_regions_scratch_bytes(1 << 16, (1 << 15) + 64, ctypes.byref(need)) == _lib.XRS_OK
    assert need.value >= 18 * (1 << 16) * ((1 << 15) + 64)
    cases = [
        (lambda: lib.xrs_zonal_regions(p, F32, 32, 4, 4, 6, p, 16, p, 1 << 20, None), b"neighborhood"),
        (lambda: lib.xrs_zonal_regions(p, 11, 32, 4, 4, 4, p, 16, p, 1 << 20, None), b"cell type"),
        (lambda: lib.xrs_zonal_regions(p, F32, 8, 4, 4, 4, p, 16, p, 1 << 20, None), b"pitch"),
        (lambda: lib.xrs_zonal_regions(p, F32, 16, 4, 4, 4, p, 16, p, 8, None), b"too small"),
        (lambda: lib.xrs_zonal_regions(None, F32, 16, 4, 4, 4, p, 16, p, 1 << 20, None), b"NULL"),
        (lambda: lib.xrs_zonal_regions(p, F32, 16, -1, 4, 4, p, 16, p, 1 << 20, None), b"negative"),
        (lambda: lib.xrs_zonal_bounds(p, F32, 16, 4, 4, 2, p, None, 1, p, None), b"mode"),
        (lambda: lib.xrs_zonal_bounds(p, 11, 16, 4, 4, 0, p, None, 1, p, None), b"cell type"),
        (lambda: lib.xrs_zonal_bounds(p, F32, 8, 4, 4, 0, p, None, 1, p, None), b"pitch"),
        (lambda: lib.xrs_zonal_bounds(p, F32, 16, 4, 4, 0, None, None, 1, p, None), b"NULL values"),
        (lambda: lib.xrs_zonal_bounds(p, F32, 16, 4, 4, 0, p, None, 1, None, None), b"NULL"),
    ]
    for call, words in cases:
        assert call() == _lib.XRS_EINVAL, words
        assert words in lib.xrs_last_error_string(), (words, lib.xrs_last_error_string())
    assert lib.xrs_zonal_regions(p, F32, 0, 0, 4, 4, p, 0, None, 0, None) == _lib.XRS_OK   # nothing to do

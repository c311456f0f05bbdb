"""viewshed: viewshed_los.cuh compiled for the host and checked against the unmodified reference's outputs and a
brute force over every cell, the argument rules, and on the GPU the reference's outputs and properties, equality
with the host build, cell types, containers and streams."""
import ctypes
import importlib
import inspect
import json
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "xarray-spatial_b200", "csrc", "viewshed_los.cuh")
GOLDEN = os.path.join(ROOT, "tests", "golden")
TIE = 1e-12   # a cell whose blocker margin is below this may flip with an ulp of atan


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(GOLDEN, "viewshed_reference.npz"), allow_pickle=False))


def _vs():
    return importlib.import_module("xrspatial_b200.viewshed")


# ----------------------------------------------------------------------------- the header on the host
@pytest.fixture(scope="module")
def host(tmp_path_factory):
    d = tmp_path_factory.mktemp("vs")
    cpp, so = str(d / "v.cpp"), str(d / "v.so")
    with open(cpp, "w") as f:
        f.write('#include "%s"\n' % HEADER + r"""
#include <vector>
using namespace xrs::vs;
struct Z {
    const double *z; int64_t W;
    double operator()(int64_t r, int64_t c) const { return z[r * W + c]; }
};
#define ARGS const double *z, int64_t H, int64_t W, int64_t vr, int64_t vc, double vp, double tg, double ew, double ns
#define VIEW View v{H, W, vr, vc, vp, tg, ew, ns}; Z zz{z, W}
extern "C" double vs_atan(double x) { return atan64(x); }
// every cell through a node table, as the kernels run
extern "C" void vs_run(ARGS, double *out) {
    VIEW;
    std::vector<Node> t(H * W);
    for (int64_t r = 0; r < H; ++r)
        for (int64_t c = 0; c < W; ++c)
            if (r != vr || c != vc) t[r * W + c] = make_node(v, zz, r, c);
    for (int64_t r = 0; r < H; ++r)
        for (int64_t c = 0; c < W; ++c)
            out[r * W + c] = cell_value(v, [&](int64_t a, int64_t b) { return t[a * W + b]; }, r, c);
}
// one cell on its own: the nodes it needs are built as the ray reaches them
extern "C" void vs_cells(ARGS, int64_t n, const int64_t *idx, double *out) {
    VIEW;
    for (int64_t k = 0; k < n; ++k)
        out[k] = cell_value(v, [&](int64_t a, int64_t b) { return make_node(v, zz, a, b); }, idx[k] / W, idx[k] % W);
}
// the brute-force margin of listed cells: the largest interpolated blocker gradient minus the target's
extern "C" void vs_margin(ARGS, int64_t n, const int64_t *idx, double *out) {
    VIEW;
    for (int64_t k = 0; k < n; ++k) {
        const int64_t r = idx[k] / W, c = idx[k] % W;
        const Node t = make_node(v, zz, r, c);
        const double kt = v.key(r, c), gt = target_grad(v, kt, t.zt), th = t.a1;
        double mx = -INFINITY;
        for (int64_t a = 0; a < H; ++a)
            for (int64_t b = 0; b < W; ++b) {
                if ((a == vr && b == vc) || !(v.key(a, b) < kt)) continue;
                const Node m = make_node(v, zz, a, b);
                double A0, A1, A2;
                if (!member(m, th, A0, A1, A2)) continue;
                const double g = interp(m, A0, A1, A2, th);
                if (g > mx) mx = g;
            }
        out[k] = mx - gt;
    }
}
// brute force over every cell: the largest interpolated blocker gradient minus the target's (-inf without one,
// NaN when the target's gradient is NaN), and whether the ray walk enumerates every blocker
extern "C" void vs_brute(ARGS, double *margin, int *superset) {
    VIEW;
    std::vector<char> seen(H * W);
    for (int64_t r = 0; r < H; ++r)
        for (int64_t c = 0; c < W; ++c) {
            const int64_t k = r * W + c;
            superset[k] = 1;
            margin[k] = -INFINITY;
            if (r == vr && c == vc) continue;
            const Node t = make_node(v, zz, r, c);
            const double kt = v.key(r, c), gt = target_grad(v, kt, t.zt), th = t.a1;
            std::fill(seen.begin(), seen.end(), 0);
            for_each_candidate(v, r - vr, c - vc, [&](int64_t a, int64_t b) { seen[a * W + b] = 1; return false; });
            double mx = -INFINITY;
            for (int64_t a = 0; a < H; ++a)
                for (int64_t b = 0; b < W; ++b) {
                    if ((a == vr && b == vc) || !(v.key(a, b) < kt)) continue;
                    const Node n = make_node(v, zz, a, b);
                    double A0, A1, A2;
                    if (!member(n, th, A0, A1, A2)) continue;
                    if (!seen[a * W + b]) superset[k] = 0;
                    const double g = interp(n, A0, A1, A2, th);
                    if (g > mx) mx = g;
                }
            margin[k] = gt == gt ? mx - gt : NAN;
        }
}
""")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, cpp])
    lib = ctypes.CDLL(so)
    I64, D, P = ctypes.c_int64, ctypes.c_double, ctypes.c_void_p
    head = [P, I64, I64, I64, I64, D, D, D, D]
    lib.vs_atan.argtypes, lib.vs_atan.restype = [D], D
    lib.vs_run.argtypes = head + [P]
    lib.vs_cells.argtypes = head + [I64, P, P]
    lib.vs_brute.argtypes = head + [P, P]
    lib.vs_margin.argtypes = head + [I64, P, P]
    return lib


class Case:
    """A viewshed call reduced to the C arguments by the package's own glue (viewshed._view)."""

    def __init__(self, z, xs, ys, x, y, obs=0, tgt=0):
        self.z, self.xs, self.ys, self.x, self.y, self.obs, self.tgt = z, xs, ys, x, y, obs, tgt
        self.view = _vs()._view(np.asarray(xs), np.asarray(ys), x, y, lambda r, c: z[r, c], obs, tgt)

    def args(self):
        z = np.ascontiguousarray(self.z, dtype=np.float64)
        self._keep = z
        return (z.ctypes.data, z.shape[0], z.shape[1]) + self.view

    def host(self, lib):
        out = np.empty(self.z.shape)
        lib.vs_run(*self.args(), out.ctypes.data)
        return out

    def brute(self, lib):
        margin = np.empty(self.z.shape)
        sup = np.empty(self.z.shape, np.int32)
        lib.vs_brute(*self.args(), margin.ctypes.data, sup.ctypes.data)
        return margin, sup.astype(bool)

    def margin(self, lib, cells):
        cells = np.ascontiguousarray(cells, np.int64)
        out = np.empty(cells.size)
        lib.vs_margin(*self.args(), cells.size, cells.ctypes.data, out.ctypes.data)
        return out

    def gpu(self, dtype=None):
        import xrspatial_b200 as xb
        z = self.z if dtype is None else self.z.astype(dtype)
        da = xb.DataArray(z, dims=("y", "x"), coords={"y": self.ys, "x": self.xs})
        return np.asarray(xb.viewshed(da, x=self.x, y=self.y, observer_elev=self.obs, target_elev=self.tgt).data)


def _doc_case(g):
    return Case(g["doc_data"], np.linspace(1, 5, 5), np.linspace(1, 4, 4), 3, 2)


def _tv_cases(g):
    xs = g["tv_coords"]
    for (obs, elev, ri, ci), out in zip(g["tv_params"], g["tv_out"]):
        a = np.zeros((5, 5), np.int64)
        a[ri, ci] = elev
        yield Case(a, xs, xs, xs[ci], xs[ri], int(obs)), out


def _flat_cases(g):
    for (obs, tgt), out in zip(g["flat_params"], g["flat_out"]):
        yield Case(np.full((5, 4), 1.3), np.arange(4) * 0.5, np.arange(5) * 1.5, 0, 0, int(obs), int(tgt)), out


def _small_cases(g, with_raises=False):
    off = g["small_off"]
    for k, (h, w) in enumerate(g["small_shape"]):
        if g["small_raises"][k] and not with_raises:
            continue
        xo, yo = int(g["small_shape"][:k, 1].sum()), int(g["small_shape"][:k, 0].sum())
        x, y, obs, tgt = g["small_params"][k]
        z = g["small_dem"][off[k]:off[k + 1]].reshape(h, w)
        case = Case(z, g["small_x"][xo:xo + w], g["small_y"][yo:yo + h], x, y, obs, tgt)
        yield case, g["small_out"][off[k]:off[k + 1]].reshape(h, w), bool(g["small_raises"][k])


# The large cases' DEMs, as oracle/make_golden_viewshed.py builds them: exact dyadic values.
LARGE = [
    ("bench", 300, 600, "bump", None, (100.0, 50.0), 1.0, 0.0, 0.0),
    ("int", 400, 400, "int", (1.0, 1.0), (200.0, 117.0), 2.5, 0.0, 0.0),
    ("corner", 256, 512, "bump", (30.0, -30.0), (30.0 * 3, -30.0 * 250), 0.0, 1.5, 0.05),
    ("edge", 500, 200, "bump", (0.5, 1.5), (0.0, 1.5 * 321), 4.0, 0.0, 0.0),
]


def _large_dem(h, w, kind):
    i = np.arange(h, dtype=np.uint64)[:, None]
    j = np.arange(w, dtype=np.uint64)[None, :]
    noise = (((i * np.uint64(7919) + j * np.uint64(104729)) * np.uint64(2654435761)) % np.uint64(1 << 32)) >> np.uint64(24)
    if kind == "int":
        return (noise % np.uint64(11)).astype(np.float64) - 5.0
    bump = (i * (np.uint64(h - 1) - i)) * (j * (np.uint64(w - 1) - j))
    return bump.astype(np.float64) * (400.0 / float((h - 1) * (h - 1) * (w - 1) * (w - 1))) + noise.astype(np.float64) / 64.0


def _large_cases(g):
    for name, h, w, kind, res, (x, y), obs, tgt, nan in LARGE:
        z = _large_dem(h, w, kind)
        if res is None:
            xs, ys = np.linspace(-180, 180, w), np.linspace(-90, 90, h)
        else:
            xs, ys = np.arange(w) * res[0], np.arange(h) * res[1]
        if nan:
            i = np.arange(h)[:, None]
            j = np.arange(w)[None, :]
            z = np.where((((i * 31 + j * 17) % 97) < int(nan * 97)) & (i % 8 != 2), np.nan, z)
        assert np.nansum(z) == g["large_%s_sum" % name][0] and np.isnan(z).sum() == g["large_%s_sum" % name][1]
        vis = np.unpackbits(g["large_%s_vis" % name])[:h * w].reshape(h, w).astype(bool)
        yield name, Case(z, xs, ys, x, y, obs, tgt), vis, g["large_%s_idx" % name], g["large_%s_ang" % name]


def _ulps(a, b):
    return np.abs(a - b) / np.spacing(np.maximum(np.abs(a), np.abs(b)))


def _check(out, ref_vis, ref_idx, ref_ang, margin_of, label):
    """Visibility equal in every cell but near-ties (listed in the message), angles within 4 ulps."""
    vis = out >= 0
    diff = np.flatnonzero(vis.ravel() != ref_vis.ravel())
    if diff.size:
        margin = margin_of(diff)
        assert np.all(np.abs(margin) < TIE), (label, diff[np.abs(margin) >= TIE], margin)
    flat = out.ravel()[ref_idx]
    both = flat >= 0
    assert np.all(_ulps(flat[both], ref_ang[both]) <= 4), (label, np.max(_ulps(flat[both], ref_ang[both])))
    return diff


def _full(case, ref, out, lib, label):
    ref = np.asarray(ref, np.float64)
    return _check(out, ref >= 0, np.flatnonzero(ref >= 0), ref.ravel()[ref.ravel() >= 0],
                  lambda d: case.margin(lib, d), label)


def _golden_cases(g):
    yield "doc", _doc_case(g), g["doc_out"]
    for k, (case, out) in enumerate(_tv_cases(g)):
        yield "tv%d" % k, case, out
    for k, (case, out) in enumerate(_flat_cases(g)):
        yield "flat%d" % k, case, out
    for k, (case, out, _) in enumerate(_small_cases(g)):
        yield "small%d" % k, case, out


def test_atan_is_within_one_ulp_of_libm(host):
    rng = np.random.default_rng(0)
    x = np.concatenate([rng.uniform(-3, 3, 20000), 10.0 ** rng.uniform(-12, 12, 20000), [0.0, -0.0, 0.4375,
                        0.6875, 1.1875, 2.4375, 1e300, -1e300, np.inf, -np.inf]])
    ours = np.array([host.vs_atan(v) for v in x])
    assert np.max(_ulps(ours, np.arctan(x))) <= 1
    assert np.isnan(host.vs_atan(np.nan))


def test_host_build_reproduces_the_reference(host, golden):
    """Every golden output: the doc example, the reference tests' fixtures and the seeded small rasters."""
    flips = []
    n = 0
    for label, case, ref in _golden_cases(golden):
        d = _full(case, ref, case.host(host), host, label)
        n += 1
        if d.size:
            flips.append((label, d.tolist()))
            assert not np.all(np.isfinite(case.z) & (case.z == np.round(case.z))), ("integer DEM flipped", label)
    assert n > 500
    assert len(flips) <= 3, flips


def test_host_build_reproduces_the_large_reference_cases(host, golden):
    for name, case, vis, idx, ang in _large_cases(golden):
        out = case.host(host)
        diff = _check(out, vis, idx, ang, lambda d: case.margin(host, d), name)
        assert diff.size <= 2, (name, diff)


def test_the_ray_walk_holds_every_blocker(host, golden):
    """For every target of the seeded small rasters, the enumeration is a superset of the brute force's blockers
    (every cell, the exact membership and key rule)."""
    n = 0
    for case, _, _ in _small_cases(golden, with_raises=True):
        _, sup = case.brute(host)
        assert sup.all(), np.argwhere(~sup)
        n += sup.size
    rng = np.random.default_rng(5)
    for k in range(60):   # anisotropic resolutions and long thin rasters
        h, w = int(rng.integers(1, 40)), int(rng.integers(1, 40))
        z = rng.normal(0, 3, (h, w))
        xs, ys = np.arange(w) * rng.choice([0.1, 1.0, -7.0]), np.arange(h) * rng.choice([0.3, 1.0, 40.0])
        case = Case(z, xs, ys, xs[rng.integers(w)], ys[rng.integers(h)], rng.choice([0.0, 3.0]))
        _, sup = case.brute(host)
        assert sup.all(), (k, np.argwhere(~sup))
        n += sup.size
    assert n > 30000


def test_nan_in_the_observer_row_gives_the_documented_result(host, golden):
    """Where the reference raised ValueError('node not found'), NaN cells are -1 and never block: the result equals
    the brute force's decision in every cell."""
    seen = 0
    for case, _, raised in _small_cases(golden, with_raises=True):
        if not raised:
            continue
        seen += 1
        out = case.host(host)
        margin, _ = case.brute(host)
        assert np.all(out[np.isnan(case.z) & (out != 180)] == -1)   # the observer is 180 even on a NaN
        decided = (out >= 0)[np.isfinite(margin)]
        assert np.array_equal(decided, (margin <= 0)[np.isfinite(margin)])
    assert seen >= 3


def test_one_row_and_one_column_rasters_match_the_reference(host):
    """The reference's resolution is NaN there, so only the observer is seen."""
    for shape in [(1, 5), (5, 1), (1, 1)]:
        z = np.arange(np.prod(shape), dtype=np.float64).reshape(shape)
        case = Case(z, np.arange(shape[1]) * 1.0, np.arange(shape[0]) * 1.0, 0.0, 0.0, 1.0)
        want = np.full(shape, -1.0)
        want[0, 0] = 180.0
        assert np.array_equal(case.host(host), want)


def test_argument_errors():
    import xrspatial_b200 as xb
    z = np.zeros((4, 5), np.float32)
    da = xb.DataArray(z, dims=("y", "x"), coords={"y": np.arange(4.0), "x": np.arange(5.0)})
    with pytest.raises(ValueError, match="x argument"):
        xb.viewshed(da, x=-1, y=0)
    with pytest.raises(ValueError, match="y argument"):
        xb.viewshed(da, x=0, y=4.5)
    fake = type("Array", (), {"__module__": "dask.array.core", "shape": (4, 5), "ndim": 2, "dtype": z.dtype})()
    with pytest.raises(NotImplementedError):
        xb.viewshed(xb.DataArray(fake, dims=("y", "x"), coords={"y": np.arange(4.0), "x": np.arange(5.0)}), 0, 0)


def test_nearest_observer_follows_xarray():
    """sel(method='nearest'): the nearest coordinate, the larger one on a tie, ascending or descending."""
    near = _vs()._nearest
    up, down = np.arange(4.0), np.arange(4.0)[::-1].copy()
    assert [near(up, v) for v in (1.5, 0.5, 2.5, -1, 4, 1.2)] == [2, 1, 3, 0, 3, 1]
    assert [near(down, v) for v in (1.5, 0.5, 2.5, -1, 4, 1.2)] == [1, 2, 0, 3, 0, 2]


def test_c_entry_point_rejects_bad_arguments():
    import xrspatial_b200 as xb
    lib = xb._lib.lib()
    need = ctypes.c_int64()
    assert lib.xrs_viewshed_scratch_bytes(100, 200, ctypes.byref(need)) == 0 and need.value == 56 * 100 * 200
    assert lib.xrs_viewshed_scratch_bytes(-1, 200, ctypes.byref(need)) == xb._lib.XRS_EINVAL
    need = ctypes.c_int64(56 * 100 * 200)
    p = ctypes.c_void_p(256)

    def call(in_dtype=0, in_pitch=800, vr=5, vc=5, out=p, out_pitch=1600, scratch=p, scratch_bytes=None, H=100):
        return lib.xrs_viewshed(p, in_dtype, in_pitch, H, 200, vr, vc, 0.0, 0.0, 1.0, 1.0, out, out_pitch, scratch,
                                need.value if scratch_bytes is None else scratch_bytes, None)
    assert call(in_pitch=796) == xb._lib.XRS_EINVAL and b"pitch" in lib.xrs_last_error_string()
    assert call(out_pitch=800) == xb._lib.XRS_EINVAL and b"pitch" in lib.xrs_last_error_string()
    assert call(out=None) == xb._lib.XRS_EINVAL and b"NULL" in lib.xrs_last_error_string()
    assert call(scratch=None) == xb._lib.XRS_EINVAL and b"scratch" in lib.xrs_last_error_string()
    assert call(scratch_bytes=need.value - 1) == xb._lib.XRS_EINVAL and b"too small" in lib.xrs_last_error_string()
    assert call(vr=100) == xb._lib.XRS_EINVAL and b"observer" in lib.xrs_last_error_string()
    assert call(vc=-1) == xb._lib.XRS_EINVAL and b"observer" in lib.xrs_last_error_string()
    assert call(in_dtype=9) == xb._lib.XRS_EINVAL and b"cell type" in lib.xrs_last_error_string()
    assert call(H=0) == xb._lib.XRS_EINVAL


def test_public_signature_equals_the_reference():
    import xrspatial_b200 as xb
    with open(os.path.join(GOLDEN, "viewshed_signature.json")) as f:
        rp = json.load(f)["viewshed"]
    mp = [(k, v.default) for k, v in inspect.signature(inspect.unwrap(xb.viewshed)).parameters.items()]
    assert [k for k, _ in rp] == [k for k, _ in mp]
    for (k, (kind, a)), (_, b) in zip(rp, mp):
        assert (kind == "callable") == (b is inspect.Parameter.empty), k
        if kind == "repr":
            assert a == repr(b), k


# ----------------------------------------------------------------------------- on the GPU
@pytest.mark.gpu
def test_gpu_reproduces_the_reference(host, golden):
    flips = 0
    for label, case, ref in _golden_cases(golden):
        out = case.gpu()
        flips += _full(case, ref, out, host, label).size
        assert np.array_equal(out, case.host(host)), label
    assert flips <= 3
    for name, case, vis, idx, ang in _large_cases(golden):
        out = case.gpu()
        assert np.array_equal(out, case.host(host)), name
        assert _check(out, vis, idx, ang, lambda d: case.margin(host, d), name).size <= 2


@pytest.mark.gpu
def test_gpu_keeps_the_reference_properties(golden):
    """test_viewshed: the observer is 180, all is visible from at or above the flat terrain, both diagonals are
    symmetric; test_viewshed_flat: the closed-form angles."""
    xs = golden["tv_coords"]
    for case, _ in _tv_cases(golden):
        out = case.gpu()
        obs, ri, ci = case.obs, int(np.argmin(np.abs(xs - case.y))), int(np.argmin(np.abs(xs - case.x)))
        elev = case.z[ri, ci]
        assert out[ri, ci] == 180
        if obs + elev >= 0 and obs >= abs(elev):
            assert (out > -1).all()
        for sub in _diagonal_blocks(ri, ci, 5, 5):
            np.testing.assert_allclose(sub[0](out), sub[0](out).T, rtol=1e-5, atol=1e-8)
            np.testing.assert_allclose(sub[1](out)[::-1], sub[1](out)[::-1].T, rtol=1e-5, atol=1e-8)
    for obs, tgt in [(5, 0), (5, 1), (2, 0), (2, 1)]:
        xs2, ys2 = np.meshgrid(np.arange(4) * 0.5, np.arange(5) * 1.5)
        case = Case(np.full((5, 4), 1.3), np.arange(4) * 0.5, np.arange(5) * 1.5, 0, 0, obs, tgt)
        out = case.gpu()
        angle = np.rad2deg(np.arctan2(np.sqrt(xs2 ** 2 + ys2 ** 2), obs - tgt))
        angle[0, 0] = out[0, 0]
        np.testing.assert_allclose(out, angle)


def _diagonal_blocks(y, x, h, w):
    h, w = h - 1, w - 1
    t = min(y, x)
    b = min(h - y, w - x)
    t2 = min(y, w - x)
    b2 = min(h - y, x)
    return [(lambda v: v[y - t:y + b + 1, x - t:x + b + 1], lambda v: v[y - t2:y + b2 + 1, x - b2:x + t2 + 1])]


@pytest.mark.gpu
def test_gpu_equals_the_host_build_bit_for_bit(host):
    rng = np.random.default_rng(11)
    for h, w, res in [(64, 64, (1.0, 1.0)), (257, 130, (0.5, 1.5)), (512, 1024, (30.0, -30.0)),
                      (1024, 1024, (10.0, 10.0))]:
        z = np.cumsum(np.cumsum(rng.normal(0, 1, (h, w)), 0), 1) * 0.05
        z[rng.random((h, w)) < 0.01] = np.nan
        xs, ys = np.arange(w) * res[0], np.arange(h) * res[1]
        r, c = int(rng.integers(h)), int(rng.integers(w))
        z[r, c] = abs(z[r, c]) if np.isfinite(z[r, c]) else 0.0
        case = Case(z, xs, ys, xs[c], ys[r], 2.0, 0.5)
        a, b = case.gpu(), case.gpu()
        assert np.array_equal(a, b)                                 # repeated calls
        assert np.array_equal(a, case.host(host)), (h, w)


@pytest.mark.gpu
def test_gpu_equals_the_host_build_on_sampled_cells_of_8192_squared(host):
    import torch
    import xrspatial_b200 as xb
    n = 8192
    g = torch.Generator(device="cuda").manual_seed(3)
    z = torch.cumsum(torch.randn((n, n), generator=g, device="cuda", dtype=torch.float64), 1)
    z = (z + torch.cumsum(torch.randn((n, n), generator=g, device="cuda", dtype=torch.float64), 0)) * 0.3
    xs, ys = np.arange(n) * 10.0, np.arange(n) * -10.0
    da = xb.DataArray(z, dims=("y", "x"), coords={"y": ys, "x": xs})
    out = xb.viewshed(da, x=xs[n // 2], y=ys[n // 3], observer_elev=300.0).data.cpu().numpy()
    zh = z.cpu().numpy()
    case = Case(zh, xs, ys, xs[n // 2], ys[n // 3], 300.0)
    idx = np.random.default_rng(4).choice(n * n, 10000, replace=False).astype(np.int64)
    ref = np.empty(idx.size)
    host.vs_cells(*case.args(), idx.size, idx.ctypes.data, ref.ctypes.data)
    assert np.array_equal(out.ravel()[idx], ref)
    assert (ref >= 0).any() and (ref < 0).any()


@pytest.mark.gpu
def test_gpu_cell_types_agree_with_float64(host):
    rng = np.random.default_rng(8)
    z = rng.integers(0, 200, (90, 120)).astype(np.float64)
    xs, ys = np.arange(120) * 2.0, np.arange(90) * 2.0
    case = Case(z, xs, ys, xs[40], ys[70], 3, 1)
    want = case.gpu()
    for dt in (np.float32, np.float64, np.int16, np.uint16, np.int32):
        assert np.array_equal(case.gpu(dt), want), dt


@pytest.mark.gpu
def test_gpu_containers_streams_and_input(host):
    import torch
    import xrspatial_b200 as xb
    rng = np.random.default_rng(9)
    z = rng.normal(0, 5, (300, 200)).astype(np.float32)
    xs, ys = np.arange(200) * 1.0, np.arange(300) * 1.0
    want = Case(z.astype(np.float64), xs, ys, 50.0, 120.0, 1.5).host(host)
    da = xb.DataArray(z, dims=("y", "x"), coords={"y": ys, "x": xs}, attrs={"unit": "m"})
    out = xb.viewshed(da, x=50.0, y=120.0, observer_elev=1.5)
    assert isinstance(out.data, np.ndarray) and out.data.dtype == np.float64 and out.attrs == {"unit": "m"}
    assert tuple(out.dims) == ("y", "x")
    assert np.array_equal(out.data, want)
    t = torch.as_tensor(z, device="cuda")
    before = t.clone()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        dv = xb.viewshed(xb.DataArray(t, dims=("y", "x"), coords={"y": ys, "x": xs}), x=50.0, y=120.0,
                         observer_elev=1.5).data
    s.synchronize()
    assert isinstance(dv, torch.Tensor) and dv.is_cuda
    assert np.array_equal(dv.cpu().numpy(), want)
    assert torch.equal(t, before)                                 # the input is never written


@pytest.mark.gpu
def test_gpu_nan_in_the_observer_row_does_not_raise(host, golden):
    seen = 0
    for case, _, raised in _small_cases(golden, with_raises=True):
        if raised:
            seen += 1
            out = case.gpu()
            assert np.all(out[np.isnan(case.z) & (out != 180)] == -1)
            assert np.array_equal(out, case.host(host))
    assert seen >= 3

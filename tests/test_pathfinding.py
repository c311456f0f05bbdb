"""a_star_search: pathfinding_grid.cuh compiled for the host -- its exact compare against rational arithmetic, and a
host search (a Dijkstra over the header's compare, then the header's walk) against the unmodified reference's
outputs -- the argument rules and the C entry points' checks; on the GPU the reference's outputs, bit equality with
the host search up to 4096^2, repeated calls, cell types, containers and streams."""
import ctypes
import importlib
import inspect
import json
import os
import subprocess
import warnings
from fractions import Fraction

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "xarray-spatial_b200", "csrc", "pathfinding_grid.cuh")
GOLDEN = os.path.join(ROOT, "tests", "golden")
SQRT2 = np.sqrt(2.0)


def _pf():
    return importlib.import_module("xrspatial_b200.pathfinding")


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(GOLDEN, "pathfinding_reference.npz"), allow_pickle=False))


# ----------------------------------------------------------------------------- the header on the host
@pytest.fixture(scope="module")
def host(tmp_path_factory):
    d = tmp_path_factory.mktemp("pf")
    cpp, so = str(d / "p.cpp"), str(d / "p.so")
    with open(cpp, "w") as f:
        f.write('#include "%s"\n' % HEADER + r"""
#include <cmath>
#include <queue>
#include <vector>
using namespace xrs::pf;
extern "C" int pf_less(int a1, int b1, int a2, int b2) { return less(Dist{a1, b1}, Dist{a2, b2}); }
static std::vector<char> mask(const double *z, int64_t n, const double *bar, int nb) {
    std::vector<char> m(n);
    for (int64_t k = 0; k < n; ++k) {
        bool ok = z[k] == z[k];
        for (int i = 0; i < nb; ++i) ok = ok && z[k] != bar[i];
        m[k] = ok;
    }
    return m;
}
// The exact field of lengths to the goal (a Dijkstra on the header's compare), then the header's walk from the
// start; out (H W float64) is NaN except along the path; field (2 H W int32) receives the field.
extern "C" void pf_search(const double *z, int64_t H, int64_t W, const double *bar, int nb, int conn, int64_t sr,
                          int64_t sc, int64_t gr, int64_t gc, double *out, int32_t *field) {
    const std::vector<char> m = mask(z, H * W, bar, nb);
    std::vector<Dist> D(H * W, unreached());
    struct Item { Dist d; int64_t k; };
    auto later = [](const Item &x, const Item &y) { return less(y.d, x.d); };
    std::priority_queue<Item, std::vector<Item>, decltype(later)> q(later);
    if (m[gr * W + gc]) { D[gr * W + gc] = Dist{0, 0}; q.push({Dist{0, 0}, gr * W + gc}); }
    while (!q.empty()) {
        const Item it = q.top(); q.pop();
        if (!same(it.d, D[it.k])) continue;
        const int64_t r = it.k / W, c = it.k % W;
        for (int k = 0; k < n_moves(conn); ++k) {
            int dy, dx; move(conn, k, dy, dx);
            const int64_t rr = r + dy, cc = c + dx;
            if (rr < 0 || rr >= H || cc < 0 || cc >= W || !m[rr * W + cc]) continue;
            const Dist nd = add_step(it.d, dy && dx);
            if (less(nd, D[rr * W + cc])) { D[rr * W + cc] = nd; q.push({nd, rr * W + cc}); }
        }
    }
    for (int64_t k = 0; k < H * W; ++k) { out[k] = NAN; field[2 * k] = D[k].a; field[2 * k + 1] = D[k].b; }
    if (!m[sr * W + sc] || !reached(D[sr * W + sc])) return;
    auto at = [&](int64_t r, int64_t c) {
        return [&, r, c](int dy, int dx) {
            const int64_t rr = r + dy, cc = c + dx;
            return (rr < 0 || rr >= H || cc < 0 || cc >= W) ? unreached() : D[rr * W + cc];
        };
    };
    int64_t r = sr, c = sc;
    double v = 0.0;
    out[r * W + c] = v;
    while (!(r == gr && c == gc)) {
        const int k = successor(D[r * W + c], conn, at(r, c));
        if (k < 0) { out[0] = INFINITY; return; }
        int dy, dx; move(conn, k, dy, dx);
        r += dy; c += dx;
        v = path_value(v, dy && dx);
        out[r * W + c] = v;
    }
}
extern "C" void pf_snap(const double *z, int64_t H, int64_t W, const double *bar, int nb, int64_t r0, int64_t c0,
                        int64_t *rr, int64_t *cc) {
    const std::vector<char> m = mask(z, H * W, bar, nb);
    int64_t best = -1, bd = 0;
    for (int64_t k = 0; k < H * W; ++k) {
        const int64_t d2 = snap_d2(k / W, k % W, r0, c0);
        if (m[k] && snap_qualifies(d2, H, W) && (best < 0 || d2 < bd)) { best = k; bd = d2; }
    }
    *rr = best < 0 ? -1 : best / W;
    *cc = best < 0 ? -1 : best % W;
}
""")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, cpp])
    lib = ctypes.CDLL(so)
    I, I64, P = ctypes.c_int, ctypes.c_int64, ctypes.c_void_p
    lib.pf_less.argtypes, lib.pf_less.restype = [I, I, I, I], I
    lib.pf_search.argtypes = [P, I64, I64, P, I, I, I64, I64, I64, I64, P, P]
    lib.pf_snap.argtypes = [P, I64, I64, P, I, I64, I64, P, P]
    return lib


def host_search(lib, z, bars, conn, s, g):
    z = np.ascontiguousarray(z, dtype=np.float64)
    b = np.ascontiguousarray(np.append(bars, 0.0), dtype=np.float64)
    out = np.empty(z.shape)
    field = np.empty(z.shape + (2,), np.int32)
    lib.pf_search(z.ctypes.data, z.shape[0], z.shape[1], b.ctypes.data, len(bars), conn, s[0], s[1], g[0], g[1],
                  out.ctypes.data, field.ctypes.data)
    assert not np.isinf(out).any(), "the walk left the field"
    return out, field


# ----------------------------------------------------------------------------- golden cases
class Surface:
    """The DataArray a golden case was made with (make_golden_pathfinding.py): create_test_raster's coordinates."""

    def __init__(self, data, ry, rx, use_attrs):
        h, w = data.shape
        self.data, self.shape, self.ndim, self.dims = data, data.shape, 2, ("y", "x")
        self.coords = {"y": np.linspace((h - 1) * ry, 0, h), "x": np.linspace(0, (w - 1) * rx, w)}
        self.attrs = {"res": (rx, ry)} if use_attrs else {}

    def __getitem__(self, k):
        return _Coord(self.coords[k])


class _Coord:
    def __init__(self, v):
        self.data = v

    def min(self):
        return _Coord(self.data.min())

    def max(self):
        return _Coord(self.data.max())

    def item(self):
        return self.data.item()


def cases(g, prefix):
    meta, pts = g[prefix + "meta"], g[prefix + "pts"]
    do, bo = g[prefix + "data_off"], g[prefix + "bar_off"]
    for i, m in enumerate(meta):
        h, w, is_int, conn, ss, sg, attrs, ws, we, a, b, uniq = (int(v) for v in m)
        z = g[prefix + "data"][do[i]:do[i + 1]].reshape(h, w)
        data = z.astype(np.int64) if is_int else z
        yield dict(data=data, surface=Surface(data, pts[i, 0], pts[i, 1], bool(attrs)),
                   start=(pts[i, 2], pts[i, 3]), goal=(pts[i, 4], pts[i, 5]),
                   barriers=g[prefix + "barriers"][bo[i]:bo[i + 1]], conn=conn, snap_start=bool(ss),
                   snap_goal=bool(sg), warned=(bool(ws), bool(we)), ab=(a, b), unique=bool(uniq),
                   out=g[prefix + "out"][do[i]:do[i + 1]].reshape(h, w), name="%s%d" % (prefix, i))


def large_cases(g):
    for kind in ("random", "maze", "dem"):
        h, w, is_int, conn, ss, sg, attrs, ws, we, a, b, uniq = (int(v) for v in g["large_%s_meta" % kind])
        if kind == "dem":
            z = g["large_dem_z"].astype(np.float64)
            z[z == -1] = np.nan
            bars = np.zeros(0)
        else:
            z = np.unpackbits(g["large_%s_bits" % kind])[:h * w].reshape(h, w).astype(np.int64)
            bars = np.array([1.0])
        out = np.full((h, w), np.nan)
        out.ravel()[g["large_%s_idx" % kind]] = g["large_%s_val" % kind]
        yield dict(data=z, surface=Surface(z, 1.0, 1.0, True), start=(float(h - 1), 0.0), goal=(0.0, float(w - 1)),
                   barriers=bars, conn=conn, snap_start=False, snap_goal=False, warned=(False, False), ab=(a, b),
                   unique=bool(uniq), out=out, name="large_" + kind)


def steps_of(out):
    """(a, b) and the ordered cells of the path in an output."""
    idx = np.flatnonzero(~np.isnan(out.ravel()))
    if idx.size == 0:
        return (-1, -1), idx
    idx = idx[np.argsort(out.ravel()[idx], kind="stable")]
    r, c = np.divmod(idx, out.shape[1])
    diag = (np.diff(r) != 0) & (np.diff(c) != 0)
    return (int((~diag).sum()), int(diag.sum())), idx


def check_against_reference(case, got):
    ref = case["out"]
    (a, b), idx = steps_of(got)
    assert (a, b) == case["ab"], case["name"]
    if a < 0:
        assert np.isnan(got).all()
        return
    H, W = got.shape
    r, c = np.divmod(idx, W)
    ok = _pf()._crossable_rule(_pf()._barrier_values(case["barriers"]))
    assert all(ok(float(case["data"][i, j])) for i, j in zip(r, c)), case["name"]
    dr, dc = np.abs(np.diff(r)), np.abs(np.diff(c))
    assert np.all(np.maximum(dr, dc) == 1), case["name"]
    if case["conn"] == 4:
        assert np.all(dr + dc == 1), case["name"]
    run = np.zeros(idx.size)
    for k in range(1, idx.size):
        run[k] = run[k - 1] + (SQRT2 if dr[k - 1] and dc[k - 1] else 1.0)
    assert np.array_equal(got.ravel()[idx], run), case["name"]
    # the endpoints are the reference's
    assert idx[0] == np.nanargmin(ref) and idx[-1] == np.nanargmax(ref), case["name"]
    if case["unique"]:
        assert np.array_equal(got, ref, equal_nan=True), case["name"]


def run_host(lib, case):
    """The package's glue (pathfinding._plan) with the host search behind it, as the GPU path runs it."""
    z = np.asarray(case["data"], dtype=np.float64)
    H, W = z.shape

    def snap(bars, r, c):
        b = np.append(bars, 0.0)
        rr, cc = ctypes.c_int64(), ctypes.c_int64()
        lib.pf_snap(np.ascontiguousarray(z).ctypes.data, H, W, b.ctypes.data, len(bars), r, c, ctypes.byref(rr),
                    ctypes.byref(cc))
        return rr.value, cc.value

    with warnings.catch_warnings(record=True) as ws:
        warnings.simplefilter("always")
        bars, cells = _pf()._plan(case["surface"], case["start"], case["goal"], case["barriers"], "x", "y",
                                  case["conn"], case["snap_start"], case["snap_goal"], lambda r, c: float(z[r, c]),
                                  snap)
    msgs = [str(w.message) for w in ws]
    warned = ("Start at a non crossable location" in msgs, "End at a non crossable location" in msgs)
    if cells is None:
        return np.full((H, W), np.nan), warned
    return host_search(lib, z, bars, case["conn"], *cells)[0], warned


# ----------------------------------------------------------------------------- CPU: the exact compare
def convergents(limit):
    """Continued-fraction convergents p / q of sqrt(2) with p, q < limit: the closest ratios there are."""
    p0, q0, p1, q1 = 1, 0, 1, 1
    out = []
    while p1 < limit and q1 < limit:
        out.append((p1, q1))
        p0, q0, p1, q1 = p1, q1, 2 * p1 + p0, 2 * q1 + q0
    return out


# sqrt(2) lies strictly between two consecutive convergents; these are 2^-200 apart
_C = [Fraction(p, q) for p, q in convergents(2 ** 110)[-2:]]


def exact_less(a1, b1, a2, b2):
    """a1 + b1 sqrt(2) < a2 + b2 sqrt(2) in rationals: da - db sqrt(2) with sqrt(2) bracketed by two convergents.
    A nonzero da - db sqrt(2) is at least 1 / (3 |db|) away from zero, far beyond the bracket's width."""
    da, db = Fraction(a1 - a2), b2 - b1
    if db == 0:
        return da < 0
    lo, hi = sorted((da - db * _C[0], da - db * _C[1]))
    assert (lo < 0) == (hi < 0)
    return hi < 0


def test_less_matches_rationals(host):
    rng = np.random.default_rng(1)
    pairs = []
    for p, q in convergents(2 ** 31):   # p - q sqrt(2) changes sign at each, ever closer to zero
        for dp in (-1, 0, 1):
            for dq in (-1, 0, 1):
                a, b = p + dp, q + dq
                if 0 <= a < 2 ** 31 - 1 and 0 <= b < 2 ** 31 - 1:
                    pairs.append(((a, 0), (0, b)))
                    pairs.append(((0, b), (a, 0)))
                    if a + 5 < 2 ** 31 - 1 and b + 7 < 2 ** 31 - 1:
                        pairs.append(((a + 5, 7), (5, b + 7)))
    for _ in range(4000):
        hi = int(rng.choice([4, 100, 2 ** 16, 2 ** 31 - 2]))
        pairs.append(tuple(tuple(int(v) for v in rng.integers(0, hi, 2)) for _ in range(2)))
    pairs += [((3, 4), (3, 4)), ((0, 0), (0, 0)), ((1, 0), (0, 1)), ((0, 1), (1, 0)), ((2, 0), (0, 1))]
    assert len(convergents(2 ** 31)) >= 20
    for (a1, b1), (a2, b2) in pairs:
        assert bool(host.pf_less(a1, b1, a2, b2)) == exact_less(a1, b1, a2, b2), ((a1, b1), (a2, b2))
        # and it is a strict order: never both ways, equal only when the pairs are
        assert not (host.pf_less(a1, b1, a2, b2) and host.pf_less(a2, b2, a1, b1))
        if (a1, b1) != (a2, b2):
            assert host.pf_less(a1, b1, a2, b2) or host.pf_less(a2, b2, a1, b1)


def test_exact_less_reference_itself():
    # the rational helper against float64 far from ties
    for a1, b1, a2, b2 in [(3, 0, 0, 2), (2, 0, 0, 2), (7, 0, 0, 5), (0, 5, 7, 0), (10, 1, 9, 2)]:
        assert exact_less(a1, b1, a2, b2) == (a1 + b1 * SQRT2 < a2 + b2 * SQRT2)


# ----------------------------------------------------------------------------- CPU: the host build vs the reference
# test_pathfinding.py's result_8_connectivity and result_4_connectivity: snap_start and snap_goal on its NaN fixture
RESULT_8 = np.array([[np.nan, np.nan, 0., np.nan], [np.nan, SQRT2, np.nan, np.nan], [np.nan, 1 + SQRT2, np.nan, np.nan],
                     [np.nan, 2 + SQRT2, np.nan, np.nan], [np.nan] * 4])
RESULT_4 = np.array([[np.nan, 1, 0., np.nan], [np.nan, 2, np.nan, np.nan], [np.nan, 3, np.nan, np.nan],
                     [np.nan, 4, np.nan, np.nan], [np.nan] * 4])


def test_host_matches_reference_fixtures(host, golden):
    fix = list(cases(golden, "fix_"))
    for case in fix:
        got, warned = run_host(host, case)
        assert warned == case["warned"], case["name"]
        check_against_reference(case, got)
    # the connectivity fixtures have unique shortest paths, so they are matched cell for cell
    for i, want in ((1, RESULT_8), (5, RESULT_4)):
        assert fix[i]["unique"] and fix[i]["snap_start"] and fix[i]["snap_goal"]
        np.testing.assert_allclose(fix[i]["out"], want, equal_nan=True)
        assert np.array_equal(run_host(host, fix[i])[0], fix[i]["out"], equal_nan=True)


def test_host_matches_reference_small(host, golden):
    n_unique = n_path = 0
    for case in cases(golden, "small_"):
        got, warned = run_host(host, case)
        assert warned == case["warned"], case["name"]
        check_against_reference(case, got)
        n_path += case["ab"][0] >= 0
        n_unique += case["unique"]
    assert n_path > 200 and n_unique > 50


def test_host_matches_reference_large(host, golden):
    for case in large_cases(golden):
        got, _ = run_host(host, case)
        check_against_reference(case, got)


def test_golden_covers_the_edges(golden):
    m = golden["small_meta"]
    # a start that snaps to nothing (NONE): no path, and no warning since the reference then reads the last cell
    assert ((m[:, 4] == 1) & (m[:, 9] < 0) & (m[:, 7] == 0)).any()
    assert ((m[:, 9] < 0) & (m[:, 7] == 0) & (m[:, 8] == 0)).any()   # an unreachable goal
    assert set(m[:, 3]) == {4, 8} and set(m[:, 2]) == {0, 1}
    assert golden["large_maze_meta"][9] + golden["large_maze_meta"][10] > 5000   # the maze's path is long


# ----------------------------------------------------------------------------- CPU: arguments and the C ABI
class _Shim:
    def __init__(self, data, dims=("y", "x")):
        self.data, self.shape, self.ndim, self.dims = data, data.shape, data.ndim, dims
        self.attrs = {"res": (1.0, 1.0)}

    def __getitem__(self, k):
        return _Coord(np.arange(self.shape[-1 if k == "x" else -2], dtype=np.float64))


def test_argument_errors():
    f = _pf().a_star_search
    z = np.zeros((4, 5))
    with pytest.raises(ValueError, match="must be 2D"):
        f(_Shim(np.zeros((2, 3, 4)), ("b", "y", "x")), (0, 0), (1, 1))
    with pytest.raises(ValueError, match=r"should be named as coordinates:\(lat, lon\)"):
        f(_Shim(z), (0, 0), (1, 1), [], "lon", "lat")
    with pytest.raises(ValueError, match="Use either 4 or 8-connectivity."):
        f(_Shim(z), (0, 0), (1, 1), connectivity=6)
    with pytest.raises(ValueError, match="start location outside the surface graph."):
        f(_Shim(z), (4, 0), (1, 1))
    with pytest.raises(ValueError, match="goal location outside the surface graph."):
        f(_Shim(z), (0, 0), (0, 5))
    with pytest.raises(NotImplementedError):
        f(type("S", (), {"data": type("Arr", (), {"__module__": "dask.array"})(), "ndim": 2, "dims": ("y", "x")})(),
          (0, 0), (0, 0))


def test_plan_warnings():
    z = np.array([[np.nan, 1.0], [1.0, 2.0]])
    s = Surface(z, 1.0, 1.0, True)
    with pytest.warns(Warning, match="Start at a non crossable location"):
        _, cells = _pf()._plan(s, (1.0, 0.0), (0.0, 1.0), [], "x", "y", 8, False, False, lambda r, c: z[r, c], None)
    assert cells is None
    with pytest.warns(Warning, match="End at a non crossable location"):
        _, cells = _pf()._plan(s, (1.0, 1.0), (0.0, 1.0), [2], "x", "y", 8, False, False, lambda r, c: z[r, c], None)
    assert cells is None


def test_signature_matches_reference():
    with open(os.path.join(GOLDEN, "pathfinding_signature.json")) as f:
        want = json.load(f)["a_star_search"]
    got = [[k, v.default] for k, v in inspect.signature(_pf().a_star_search).parameters.items()]
    assert [k for k, _ in got] == [k for k, _ in want]
    for (k, d), (_, (kind, val)) in zip(got, want):
        if kind == "callable":
            assert d is inspect.Parameter.empty, k
        else:
            assert repr(d) == val, k
    import xrspatial_b200
    assert xrspatial_b200.a_star_search is _pf().a_star_search


def _lib():
    lib = importlib.import_module("xrspatial_b200._lib")
    try:
        lib.lib()
    except lib.XrsError:
        pytest.skip("libxrs_b200.so not built")
    return lib


def test_c_entry_points_check_arguments():
    L = _lib()
    P = ctypes.c_void_p
    fake = P(4096)   # never dereferenced: every call below fails its checks first
    n = ctypes.c_int64()
    rr, cc = ctypes.c_int64(), ctypes.c_int64()

    def search(**kw):
        a = dict(inp=fake, dt=1, pitch=80, H=4, W=10, bars=None, nb=0, conn=8, sr=0, sc=0, gr=3, gc=9, out=fake,
                 op=80, scr=fake, sb=1 << 20)
        a.update(kw)
        return L.lib().xrs_a_star_search(a["inp"], a["dt"], a["pitch"], a["H"], a["W"], a["bars"], a["nb"],
                                         a["conn"], a["sr"], a["sc"], a["gr"], a["gc"], a["out"], a["op"],
                                         a["scr"], a["sb"], None, None)

    def msg():
        return L.lib().xrs_last_error_string().decode()

    assert L.lib().xrs_a_star_scratch_bytes(4, 10, None) == L.XRS_EINVAL
    assert L.lib().xrs_a_star_scratch_bytes(0, 10, ctypes.byref(n)) == L.XRS_EINVAL
    assert L.lib().xrs_a_star_scratch_bytes(1 << 16, 1 << 15, ctypes.byref(n)) == L.XRS_EINVAL
    assert "2^31" in msg()
    assert L.lib().xrs_a_star_scratch_bytes(32768, 32768, ctypes.byref(n)) == L.XRS_OK   # 2^30 cells
    assert 9 * 2 ** 30 <= n.value < 9.1 * 2 ** 30
    assert L.lib().xrs_a_star_scratch_bytes(4, 10, ctypes.byref(n)) == L.XRS_OK
    assert search(inp=None) == L.XRS_EINVAL and "NULL input" in msg()
    assert search(out=None) == L.XRS_EINVAL and "NULL output" in msg()
    assert search(scr=None) == L.XRS_EINVAL and "NULL scratch" in msg()
    assert search(nb=2) == L.XRS_EINVAL and "barrier" in msg()
    assert search(conn=6) == L.XRS_EINVAL and "connectivity" in msg()
    assert search(dt=9) == L.XRS_EINVAL and "cell type" in msg()
    assert search(pitch=72) == L.XRS_EINVAL and "input pitch" in msg()
    assert search(op=72) == L.XRS_EINVAL and "output pitch" in msg()
    assert search(sr=4) == L.XRS_EINVAL and "start outside" in msg()
    assert search(gc=-1) == L.XRS_EINVAL and "goal outside" in msg()
    assert search(sb=n.value - 1) == L.XRS_EINVAL and "too small" in msg()
    assert search(H=1 << 16, W=1 << 15, pitch=8 << 15, op=8 << 15) == L.XRS_EINVAL and "2^31" in msg()
    snap = L.lib().xrs_a_star_snap
    assert snap(fake, 1, 80, 4, 10, None, 0, 0, 0, None, ctypes.byref(cc), fake, 256, None) == L.XRS_EINVAL
    assert snap(fake, 1, 80, 4, 10, None, 0, 4, 0, ctypes.byref(rr), ctypes.byref(cc), fake, 256,
                None) == L.XRS_EINVAL and "outside" in msg()
    assert snap(fake, 1, 80, 4, 10, None, 0, 0, 0, ctypes.byref(rr), ctypes.byref(cc), fake, 255,
                None) == L.XRS_EINVAL and "256 bytes" in msg()
    assert snap(fake, 1, 80, 4, 10, None, 0, 0, 0, ctypes.byref(rr), ctypes.byref(cc), None, 256,
                None) == L.XRS_EINVAL and "NULL scratch" in msg()


# ----------------------------------------------------------------------------- GPU
def _xb():
    return importlib.import_module("xrspatial_b200")


def gpu_call(case, data=None, **kw):
    xb = _xb()
    s = case["surface"]
    d = case["data"] if data is None else data
    agg = xb.DataArray(d, coords={"y": s.coords["y"], "x": s.coords["x"]}, dims=("y", "x"), attrs=s.attrs)
    with warnings.catch_warnings(record=True) as ws:
        warnings.simplefilter("always")
        out = xb.a_star_search(agg, case["start"], case["goal"], list(case["barriers"]), "x", "y", case["conn"],
                               case["snap_start"], case["snap_goal"], **kw)
    msgs = [str(w.message) for w in ws]
    return out, ("Start at a non crossable location" in msgs, "End at a non crossable location" in msgs)


@pytest.mark.gpu
def test_gpu_matches_reference(golden):
    for prefix in ("fix_", "small_"):
        for case in cases(golden, prefix):
            out, warned = gpu_call(case)
            assert warned == case["warned"], case["name"]
            assert out.dims == ("y", "x") and out.attrs == case["surface"].attrs
            check_against_reference(case, np.asarray(out.data))
    for case in large_cases(golden):
        check_against_reference(case, np.asarray(gpu_call(case)[0].data))


def _obstacles(rng, h, w, dens):
    z = (rng.random((h, w)) < dens).astype(np.float64)
    return z


def _maze(h, w):
    z = np.zeros((h, w))
    for i, r in enumerate(range(2, h - 1, 4)):
        z[r, :] = 1
        z[r, (w - 2, w - 1) if i % 2 == 0 else (0, 1)] = 0
    return z


def _device_search(z, bars, conn, s, g):
    import torch
    L = _lib()
    t = torch.from_numpy(np.ascontiguousarray(z)).cuda()
    b = torch.as_tensor(np.append(bars, 0.0)).cuda()
    H, W = z.shape
    n = ctypes.c_int64()
    L.call("xrs_a_star_scratch_bytes", H, W, ctypes.byref(n))
    scr = torch.empty(n.value, dtype=torch.uint8, device="cuda")
    out = torch.empty((H, W), dtype=torch.float64, device="cuda")
    rounds = ctypes.c_int64()
    L.call("xrs_a_star_search", ctypes.c_void_p(t.data_ptr()), 1, W * 8, H, W, ctypes.c_void_p(b.data_ptr()),
           len(bars), conn, s[0], s[1], g[0], g[1], ctypes.c_void_p(out.data_ptr()), W * 8,
           ctypes.c_void_p(scr.data_ptr()), n.value, ctypes.byref(rounds), None)
    field = scr[256:256 + H * W * 8].view(torch.int32).reshape(H, W, 2).cpu().numpy()
    return out.cpu().numpy(), field, rounds.value


@pytest.mark.gpu
def test_gpu_equals_host_build(host):
    rng = np.random.default_rng(5)
    shapes = [(1, 1), (1, 70), (70, 1), (33, 65), (64, 64), (100, 257), (257, 100), (511, 513), (1024, 1024)]
    for i, (h, w) in enumerate(shapes * 2):
        conn = (8, 4)[i % 2]
        dens = [0.0, 0.1, 0.3, 0.42][i % 4]
        z = _obstacles(rng, h, w, dens)
        s = (int(rng.integers(h)), int(rng.integers(w)))
        g = (int(rng.integers(h)), int(rng.integers(w)))
        if i % 3 == 0:
            s, g = (0, 0), (h - 1, w - 1)
        z[s] = z[g] = 0
        want, wf = host_search(host, z, [1.0], conn, s, g)
        got, gf, _ = _device_search(z, [1.0], conn, s, g)
        assert np.array_equal(gf, wf), (h, w, conn)
        assert np.array_equal(got, want, equal_nan=True), (h, w, conn)


@pytest.mark.gpu
def test_gpu_equals_host_build_large(host):
    rng = np.random.default_rng(6)
    for z, conn in ((_obstacles(rng, 4096, 4096, 0.3), 8), (_maze(2048, 2048), 8), (_maze(2048, 2048), 4)):
        H, W = z.shape
        z[0, 0] = z[H - 1, W - 1] = 0
        want, wf = host_search(host, z, [1.0], conn, (0, 0), (H - 1, W - 1))
        got, gf, rounds = _device_search(z, [1.0], conn, (0, 0), (H - 1, W - 1))
        assert np.array_equal(gf, wf)
        assert np.array_equal(got, want, equal_nan=True)
        assert rounds > 0
        again, gf2, _ = _device_search(z, [1.0], conn, (0, 0), (H - 1, W - 1))
        assert np.array_equal(again, got, equal_nan=True) and np.array_equal(gf2, gf)


@pytest.mark.gpu
def test_gpu_snap_matches_host(host):
    import torch
    L = _lib()
    rng = np.random.default_rng(8)
    for h, w in ((1, 1), (3, 7), (40, 33), (300, 200)):
        for dens in (0.5, 0.97, 1.0):
            z = _obstacles(rng, h, w, dens)
            t = torch.from_numpy(z).cuda()
            b = torch.tensor([1.0, 0.0], dtype=torch.float64, device="cuda")
            scr = torch.empty(256, dtype=torch.uint8, device="cuda")
            for _ in range(5):
                r0, c0 = int(rng.integers(h)), int(rng.integers(w))
                rr, cc, hr, hc = ctypes.c_int64(), ctypes.c_int64(), ctypes.c_int64(), ctypes.c_int64()
                L.call("xrs_a_star_snap", ctypes.c_void_p(t.data_ptr()), 1, w * 8, h, w, ctypes.c_void_p(b.data_ptr()),
                       1, r0, c0, ctypes.byref(rr), ctypes.byref(cc), ctypes.c_void_p(scr.data_ptr()), 256, None)
                zz = np.ascontiguousarray(z)
                bb = np.array([1.0, 0.0])
                host.pf_snap(zz.ctypes.data, h, w, bb.ctypes.data, 1, r0, c0, ctypes.byref(hr), ctypes.byref(hc))
                assert (rr.value, cc.value) == (hr.value, hc.value), (h, w, dens, r0, c0)


def _one(z, barriers=(1,), shape_of=None):
    """A corner-to-corner case on z (numpy, or any container with `shape_of` the numpy raster it holds)."""
    zs = np.asarray(z if shape_of is None else shape_of)
    h, w = zs.shape
    return dict(data=z, surface=Surface(zs, 1.0, 1.0, True), start=(float(h - 1), 0.0), goal=(0.0, float(w - 1)),
                barriers=np.asarray(barriers, np.float64), conn=8, snap_start=False, snap_goal=False)


@pytest.mark.gpu
def test_gpu_cell_types_agree_with_float64():
    import torch
    rng = np.random.default_rng(11)
    z = rng.integers(0, 4, (130, 90))
    z[-1, 0] = z[0, -1] = 2
    case = _one(z.astype(np.float64), barriers=(1, 3))
    want = np.asarray(gpu_call(case)[0].data)
    assert not np.isnan(want).all()
    for dt in (np.float32, np.int32, np.int64, np.int16, np.uint16, np.uint8, np.int8, np.bool_):
        zz = (z % 2 if dt == np.bool_ else z).astype(dt)
        c = _one(zz, barriers=(1, 3))
        if dt == np.bool_:
            c["barriers"] = np.array([1.0])
            w2 = np.asarray(gpu_call(_one((z % 2).astype(np.float64), barriers=(1,)))[0].data)
            assert np.array_equal(np.asarray(gpu_call(c)[0].data), w2, equal_nan=True)
            continue
        assert np.array_equal(np.asarray(gpu_call(c)[0].data), want, equal_nan=True), dt
    for dt in (torch.float32, torch.int32, torch.int64, torch.int16, torch.float64):
        c = _one(torch.from_numpy(z).to(dt).cuda(), barriers=(1, 3), shape_of=z)
        assert np.array_equal(gpu_call(c)[0].data.cpu().numpy(), want, equal_nan=True), dt


@pytest.mark.gpu
def test_gpu_containers_streams_views():
    import torch
    rng = np.random.default_rng(12)
    z = _obstacles(rng, 200, 300, 0.25)
    z[-1, 0] = z[0, -1] = 0
    case = _one(z)
    want = np.asarray(gpu_call(case)[0].data)
    assert isinstance(want, np.ndarray) and not np.isnan(want).all()
    t = torch.from_numpy(z).cuda()
    keep = t.clone()
    out = gpu_call(case, data=t)[0].data
    assert isinstance(out, torch.Tensor) and out.is_cuda and out.dtype == torch.float64
    assert np.array_equal(out.cpu().numpy(), want, equal_nan=True)
    assert torch.equal(t, keep)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        out = gpu_call(case, data=t)[0].data
    s.synchronize()
    assert np.array_equal(out.cpu().numpy(), want, equal_nan=True)
    big = torch.zeros((200, 600), dtype=torch.float64, device="cuda")
    big[:, ::2] = t
    view = big[:, ::2]
    assert view.stride(1) == 2
    assert np.array_equal(gpu_call(case, data=view)[0].data.cpu().numpy(), want, equal_nan=True)
    zc = z.copy()
    gpu_call(case, data=zc)
    assert np.array_equal(zc, z)
    a = gpu_call(case)[0].data
    b = gpu_call(case)[0].data
    assert np.array_equal(a, b, equal_nan=True)


@pytest.mark.gpu
def test_gpu_reference_test_properties():
    # test_a_star_search_no_barriers: from any start to any goal, 0 at the start and a positive maximum elsewhere
    data = np.array([[0, 1, 0, 0], [1, 1, 0, 0], [0, 1, 2, 2], [1, 0, 2, 0], [0, 2, 2, 2]])
    xb = _xb()
    agg = xb.DataArray(data, coords={"lat": np.linspace(2.0, 0, 5), "lon": np.linspace(0, 1.5, 4)},
                       dims=("lat", "lon"), attrs={"res": (0.5, 0.5)})
    for y0 in agg["lat"].data:
        for x0 in agg["lon"].data:
            for y1 in agg["lat"].data[::2]:
                for x1 in agg["lon"].data[::3]:
                    out = np.asarray(xb.a_star_search(agg, (y0, x0), (y1, x1), [], "lon", "lat").data)
                    assert out.dtype == np.float64 and np.nanmin(out) == 0
                    assert (np.nanmax(out) == 0) == ((y0, x0) == (y1, x1))

"""proximity, allocation and direction: the column pass of proximity_envelope.cuh compiled for the host and checked
against a float64 brute force, the argument rules, and on the GPU the reference's tables, a row-major brute force,
the reference's own outputs, SciPy's exact transform at scale and independence from the band split."""
import ctypes
import json
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "xarray-spatial_b200", "csrc", "proximity_envelope.cuh")
GOLDEN = os.path.join(ROOT, "tests", "golden")
METRICS = {"EUCLIDEAN": 0, "GREAT_CIRCLE": 1, "MANHATTAN": 2}
RAD = np.pi / 180.0


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(GOLDEN, "proximity_reference.npz"), allow_pickle=False))


# ----------------------------------------------------------------------------- float64 statements of the kernels
def _tables(xs, ys):
    return np.cos(ys * RAD), np.sin(ys * RAD), xs * RAD


def _pair_cost(metric, xs, ys, ti, tc, ci, cc):
    """The float64 key the kernels minimise between cells (ci, cc) and targets (ti, tc) (broadcasting)."""
    if metric == 1:
        cosl, sinl, lam = _tables(xs, ys)
        v = cosl[ti] * np.cos(lam[tc] - lam[cc])
        return -(cosl[ci] * v + sinl[ci] * sinl[ti])
    dx = xs[tc] - xs[cc]
    dy = ys[ti] - ys[ci]
    return dx * dx + dy * dy if metric == 0 else np.abs(dx) + np.abs(dy)


def _row_pass(mask, xs, metric):
    """Each cell's pick within its own row: the nearer of the last target at or before it and the first at or after
    it (the great circle adds the row's first and last target); the earlier column on a tie; -1 without one."""
    H, W = mask.shape
    lam = xs * RAD
    ridx = np.full((H, W), -1, np.int32)
    cols = np.arange(W)
    for r in range(H):
        t = np.flatnonzero(mask[r])
        if t.size == 0:
            continue
        k = np.searchsorted(t, cols, side="right")
        left = np.where(k > 0, t[np.maximum(k - 1, 0)], -1)
        k2 = np.searchsorted(t, cols, side="left")
        right = np.where(k2 < t.size, t[np.minimum(k2, t.size - 1)], -1)
        cands = [left, right] if metric != 1 else [np.full(W, t[0]), left, right, np.full(W, t[-1])]
        best = np.full(W, -1)
        bk = np.full(W, np.inf)
        for cnd in cands:
            ok = cnd >= 0
            c_safe = np.where(ok, cnd, 0)
            if metric == 1:
                key = -np.cos(lam[c_safe] - lam)
            else:
                dx = xs[c_safe] - xs
                key = dx * dx if metric == 0 else np.abs(dx)
            better = ok & ((best < 0) | (key < bk))
            best = np.where(better, cnd, best)
            bk = np.where(better, key, bk)
        ridx[r] = np.where(mask[r], cols, best)   # a target keeps itself
    return ridx


def _brute(mask, xs, ys, metric):
    """(row, col) of the nearest target of every cell under the kernels' float64 key, the first in row-major order
    among equal keys, and that key; -1 where there is no target."""
    H, W = mask.shape
    ti, tc = np.nonzero(mask)
    rows = np.full((H, W), -1)
    cols = np.full((H, W), -1)
    best = np.full((H, W), np.inf)
    if ti.size == 0:
        return rows, cols, best
    ci, cc = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    ci, cc = ci.ravel(), cc.ravel()
    for s in range(0, ci.size, 4096):
        a, b = ci[s:s + 4096, None], cc[s:s + 4096, None]
        cost = _pair_cost(metric, xs, ys, ti[None, :], tc[None, :], a, b)
        k = np.argmin(cost, axis=1)
        rows.ravel()[s:s + 4096] = ti[k]
        cols.ravel()[s:s + 4096] = tc[k]
        best.ravel()[s:s + 4096] = cost[np.arange(k.size), k]
    return rows, cols, best


def _outputs(data, xs, ys, rows, cols, metric, mode, max_distance=np.inf):
    """The reference's output values for a given nearest target (proximity.py:222-258 and its float32 steps)."""
    H, W = data.shape
    out = np.full((H, W), np.nan, np.float32)
    ii, cc = np.nonzero(rows >= 0)
    r, t = rows[ii, cc], cols[ii, cc]
    xt, yt, xc, yc = xs[t], ys[r], xs[cc], ys[ii]
    if metric == 0:
        d = np.sqrt((xt - xc) ** 2 + (yt - yc) ** 2)
    elif metric == 2:
        d = np.abs(xt - xc) + np.abs(yt - yc)
    else:
        lat1, lon1, lat2, lon2 = yt * RAD, xt * RAD, yc * RAD, xc * RAD
        a = np.sin((lat2 - lat1) / 2.0) ** 2 + np.cos(lat1) * np.cos(lat2) * np.sin((lon2 - lon1) / 2.0) ** 2
        d = 6378137.0 * 2 * np.arcsin(np.sqrt(a))
    f = d.astype(np.float32)
    sq = (f * f).astype(np.float32)
    keep = (float(max_distance) ** 2 >= sq.astype(np.float64)) | ((r == ii) & (t == cc))
    if mode == 0:
        val = np.sqrt(sq.astype(np.float64)).astype(np.float32)
    elif mode == 1:
        val = data[r, t].astype(np.float32)
    else:
        x, y = xt - xc, yt - yc
        dd = np.arctan2(-y, x) * 57.29578
        dd = np.where(dd < 0, 90.0 - dd, np.where(dd > 90.0, 360.0 - dd + 90.0, 90.0 - dd))
        val = np.where((x == 0) & (y == 0), 0.0, dd).astype(np.float32)
    out[ii[keep], cc[keep]] = val[keep]
    return out


# ----------------------------------------------------------------------------- the column pass on the host
@pytest.fixture(scope="module")
def column_pass(tmp_path_factory):
    d = tmp_path_factory.mktemp("prox")
    cpp, so = str(d / "c.cpp"), str(d / "c.so")
    with open(cpp, "w") as f:
        f.write('#include "%s"\n' % HEADER + r"""
#include <vector>
using namespace xrs::prox;
template <int M> static void run(int64_t H, int64_t W, const int32_t *ridx, const double *X, const double *Y,
                                 const double *cosl, const double *sinl, const double *lam, int64_t band_rows,
                                 int32_t *out) {
    const int nb = (int)((H + band_rows - 1) / band_rows);
    std::vector<int32_t> stk(H * W), blo(nb * W), bhi(nb * W), bprev(nb * W), boff((nb + 1) * W);
    Column<M> col;
    col.ridx = ridx; col.stk = stk.data(); col.blo = blo.data(); col.bhi = bhi.data(); col.bprev = bprev.data();
    col.boff = boff.data(); col.X = X; col.Y = Y; col.cosl = cosl; col.sinl = sinl; col.lam = lam;
    col.H = H; col.W = W; col.band_rows = band_rows; col.nb = nb;
    for (int64_t c = 0; c < W; ++c) { col.c = c; for (int b = 0; b < nb; ++b) build_band(col, b); }
    for (int64_t c = 0; c < W; ++c) { col.c = c; merge_bands(col); }
    for (int64_t c = 0; c < W; ++c) {
        col.c = c;
        for (int b = 0; b < nb; ++b) query_band(col, b, [&](int64_t i, int64_t r) { out[i * W + c] = (int32_t)r; });
    }
}
extern "C" void column_pass(int metric, int64_t H, int64_t W, const int32_t *ridx, const double *X, const double *Y,
                            const double *cosl, const double *sinl, const double *lam, int64_t band_rows,
                            int32_t *out) {
    if (metric == 0) run<0>(H, W, ridx, X, Y, cosl, sinl, lam, band_rows, out);
    else if (metric == 1) run<1>(H, W, ridx, X, Y, cosl, sinl, lam, band_rows, out);
    else run<2>(H, W, ridx, X, Y, cosl, sinl, lam, band_rows, out);
}
""")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, cpp])
    lib = ctypes.CDLL(so)
    P = ctypes.c_void_p
    lib.column_pass.argtypes = [ctypes.c_int, ctypes.c_int64, ctypes.c_int64, P, P, P, P, P, P, ctypes.c_int64, P]

    def call(mask, xs, ys, metric, band_rows):
        H, W = mask.shape
        ridx = _row_pass(mask, xs, metric)
        cosl, sinl, lam = _tables(xs, ys)
        out = np.empty((H, W), np.int32)
        arrs = [np.ascontiguousarray(a) for a in (ridx, xs, ys, cosl, sinl, lam)]
        lib.column_pass(metric, H, W, *[a.ctypes.data for a in arrs], band_rows, out.ctypes.data)
        rows = out.astype(np.int64)
        cols = np.where(rows >= 0, ridx[np.maximum(rows, 0), np.arange(W)[None, :]], -1)
        return rows, cols
    return call


def _random_case(rng, metric, integer):
    H, W = int(rng.integers(1, 48)), int(rng.integers(1, 48))
    mask = rng.random((H, W)) < rng.choice([0.005, 0.03, 0.1, 0.4, 1.0])
    if metric == 1:
        span = rng.choice([60.0, 358.0])
        xs = np.linspace(-span / 2, span / 2, W) if integer else np.sort(rng.uniform(-179.9, 179.9, W))
        ys = np.linspace(-80, 80, H) if not integer else np.arange(H) - H // 2.0
    elif integer:
        xs, ys = np.arange(W) * rng.choice([1.0, 30.0]), np.arange(H) * rng.choice([1.0, 30.0, 2.0])
    else:
        xs, ys = np.cumsum(rng.uniform(0.3, 3.0, W)), np.cumsum(rng.uniform(0.3, 3.0, H)) * 0.7
    if rng.random() < 0.5:
        ys = ys[::-1].copy()
    if rng.random() < 0.3:
        xs = xs[::-1].copy()
    return mask, xs.astype(np.float64), ys.astype(np.float64)


@pytest.mark.parametrize("metric", [0, 2, 1])
def test_column_pass_on_the_host_equals_the_brute_force(column_pass, metric):
    """Envelope, band merge and walk compiled with g++ from the shipped header, on random target sets: integer
    grids pick exactly the brute force's target (row-major first among equal keys); other coordinates pick a
    target whose key equals the minimum to rounding.  Every band split gives the same picks."""
    rng = np.random.default_rng(100 + metric)
    for case in range(120):
        integer = case % 2 == 0
        mask, xs, ys = _random_case(rng, metric, integer)
        rows, cols = column_pass(mask, xs, ys, metric, 1 << 20)
        br, bc, best = _brute(mask, xs, ys, metric)
        assert np.array_equal(rows >= 0, br >= 0)
        m = rows >= 0
        ii, cc = np.nonzero(m)
        got = _pair_cost(metric, xs, ys, rows[m], cols[m], ii, cc)
        if integer and metric != 1:
            assert np.array_equal(rows, br) and np.array_equal(cols, bc), case
        else:
            np.testing.assert_allclose(got, best[m], rtol=1e-12, atol=1e-12 * np.abs(best[m]).max(initial=1.0))
        for band_rows in (1, 2, 3, 7, 16):
            r2, c2 = column_pass(mask, xs, ys, metric, band_rows)
            assert np.array_equal(r2, rows) and np.array_equal(c2, cols), (case, band_rows)


def test_great_circle_column_pass_crosses_the_antimeridian(column_pass):
    """A target just east of -180 is the nearest one of cells just west of +180."""
    xs = np.linspace(-179.0, 179.0, 180)
    ys = np.linspace(-30.0, 30.0, 13)
    mask = np.zeros((13, 180), bool)
    mask[6, 0] = True
    mask[2, 90] = True
    rows, cols = column_pass(mask, xs, ys, 1, 4)
    assert cols[6, 179] == 0 and rows[6, 179] == 6
    br, bc, _ = _brute(mask, xs, ys, 1)
    assert np.array_equal(cols, bc) and np.array_equal(rows, br)


# ----------------------------------------------------------------------------- host-side API rules
def test_scalar_distances_equal_the_reference(golden):
    import xrspatial_b200 as xb
    for p, (e, m, g) in zip(golden["scalar_points"], golden["scalar_values"]):
        assert xb.euclidean_distance(*p) == pytest.approx(e, rel=1e-15)
        assert xb.manhattan_distance(*p) == pytest.approx(m, rel=1e-15)
        assert xb.great_circle_distance(*p) == pytest.approx(g, rel=1e-13, abs=1e-9)
    for x, y in zip([-181, 181, 0, 0], [0, 0, -91, 91]):
        with pytest.raises(ValueError):
            xb.great_circle_distance(x1=0, x2=x, y1=0, y2=y)


def _da(data, xs, ys, dims=("y", "x")):
    import xrspatial_b200 as xb
    return xb.DataArray(data, dims=dims, coords={dims[0]: ys, dims[1]: xs}, attrs={"res": (1.0, 1.0)})


def test_argument_errors():
    import xrspatial_b200 as xb
    z = np.zeros((4, 5), np.float32)
    with pytest.raises(ValueError, match="should be named"):
        xb.proximity(_da(z, np.arange(5.0), np.arange(4.0), dims=("lat", "lon")))
    with pytest.raises(ValueError):
        xb.proximity(_da(z, np.arange(5.0) * 50, np.arange(4.0)), distance_metric="GREAT_CIRCLE")
    with pytest.raises(ValueError):
        xb.allocation(_da(z, np.arange(5.0), np.arange(4.0) * 40), distance_metric="GREAT_CIRCLE")
    with pytest.raises(NotImplementedError, match="strictly ascending or descending"):
        xb.direction(_da(z, np.array([0.0, 1.0, 3.0, 2.0, 4.0]), np.arange(4.0)))
    with pytest.raises(NotImplementedError):
        xb.proximity(_da(z, np.arange(5.0), np.array([0.0, 1.0, 1.0, 2.0])))


def test_c_entry_point_rejects_bad_arguments():
    import xrspatial_b200 as xb
    lib = xb._lib.lib()
    need = ctypes.c_int64()
    assert lib.xrs_proximity_scratch_bytes(100, 200, 0, ctypes.byref(need)) == 0 and need.value >= 8 * 100 * 200
    p = ctypes.c_void_p(256)

    def call(in_pitch=800, out=p, out_pitch=800, scratch_bytes=None):
        return lib.xrs_proximity(p, 0, in_pitch, 100, 200, p, p, None, 0, 1.0, 0, 0, out, out_pitch, p,
                                 need.value if scratch_bytes is None else scratch_bytes, 0, None)
    assert call(in_pitch=796) == xb._lib.XRS_EINVAL and b"pitch" in lib.xrs_last_error_string()
    assert call(out_pitch=6) == xb._lib.XRS_EINVAL and b"pitch" in lib.xrs_last_error_string()
    assert call(out=None) == xb._lib.XRS_EINVAL and b"NULL" in lib.xrs_last_error_string()
    assert call(scratch_bytes=need.value - 1) == xb._lib.XRS_EINVAL and b"too small" in lib.xrs_last_error_string()


def test_public_signatures_equal_the_reference():
    import importlib
    import inspect
    px = importlib.import_module("xrspatial_b200.proximity")   # the package's `proximity` is the function
    with open(os.path.join(GOLDEN, "proximity_signatures.json")) as f:
        table = json.load(f)
    assert sorted(table) == sorted(["proximity", "allocation", "direction", "euclidean_distance",
                                    "manhattan_distance", "great_circle_distance"])
    for n, rp in table.items():
        mp = [(k, v.default) for k, v in inspect.signature(inspect.unwrap(getattr(px, n))).parameters.items()]
        assert [k for k, _ in rp] == [k for k, _ in mp], n
        for (k, (kind, a)), (_, b) in zip(rp, mp):
            assert (kind == "callable") == (b is inspect.Parameter.empty) or a == repr(b), (n, k)
            if kind == "repr":
                assert a == repr(b), (n, k)


# ----------------------------------------------------------------------------- GPU
def _run(data, xs, ys, metric, mode, target_values=(), max_distance=np.inf, band_rows=0):
    import importlib
    px = importlib.import_module("xrspatial_b200.proximity")
    name = [k for k, v in METRICS.items() if v == metric][0]
    return px._process(_da(data, xs, ys), "x", "y", list(target_values), max_distance, name, mode, band_rows)


def _ulp_close(got, want):
    assert np.array_equal(np.isnan(got), np.isnan(want))
    m = ~np.isnan(want)
    assert (np.abs(got[m] - want[m]) <= np.spacing(np.abs(want[m]).astype(np.float32))).all()


@pytest.mark.gpu
def test_reference_tables(golden):
    import xrspatial_b200 as xb
    data, lon, lat = golden["table_data"], golden["table_lon"], golden["table_lat"]
    agg = xb.DataArray(data, dims=["lat", "lon"], coords={"lat": lat, "lon": lon}, attrs={"unit": "m"})
    kw = dict(x="lon", y="lat")
    checks = [
        (xb.proximity(agg, **kw), golden["table_result_default_proximity"]),
        (xb.proximity(agg, target_values=list(golden["table_result_target_proximity__param"]), **kw),
         golden["table_result_target_proximity"]),
        (xb.proximity(agg, distance_metric="MANHATTAN", **kw), golden["table_result_manhattan_proximity"]),
        (xb.proximity(agg, distance_metric="GREAT_CIRCLE", **kw), golden["table_result_great_circle_proximity"]),
        (xb.proximity(agg, max_distance=float(golden["table_result_max_distance_proximity__param"]), **kw),
         golden["table_result_max_distance_proximity"]),
        (xb.allocation(agg, **kw), golden["table_result_default_allocation"]),
        (xb.allocation(agg, max_distance=float(golden["table_result_max_distance_allocation__param"]), **kw),
         golden["table_result_max_distance_allocation"]),
        (xb.direction(agg, **kw), golden["table_result_default_direction"]),
        (xb.direction(agg, max_distance=float(golden["table_result_max_distance_direction__param"]), **kw),
         golden["table_result_max_distance_direction"]),
    ]
    for got, want in checks:
        assert isinstance(got.data, np.ndarray) and got.data.dtype == np.float32
        assert tuple(got.dims) == ("lat", "lon") and got.attrs == {"unit": "m"}
        np.testing.assert_allclose(got.data, want, rtol=1e-5, equal_nan=True)
    q = xb.DataArray(golden["qgis_data"], dims=["y", "x"], coords={"y": golden["qgis_y"], "x": golden["qgis_x"]})
    got = xb.proximity(q, target_values=list(golden["table_qgis_proximity_distance_target_values__param"]))
    np.testing.assert_allclose(got.data, golden["table_qgis_proximity_distance_target_values"], rtol=1e-5,
                               equal_nan=True)


@pytest.mark.gpu
def test_containers():
    import torch
    import xrspatial_b200 as xb
    rng = np.random.default_rng(3)
    z = (rng.random((37, 53)) < 0.05).astype(np.float32)
    xs, ys = np.arange(53.0), np.arange(37.0)[::-1]
    host = xb.proximity(_da(z, xs, ys)).data
    dev = xb.proximity(_da(torch.from_numpy(z).cuda(), xs, ys)).data
    assert isinstance(dev, torch.Tensor) and dev.is_cuda and dev.dtype == torch.float32
    assert np.array_equal(dev.cpu().numpy(), host, equal_nan=True)
    ds = xb.Dataset({"a": _da(z, xs, ys), "b": _da(z * 2, xs, ys)})
    out = xb.allocation(ds)
    assert isinstance(out, xb.Dataset)
    np.testing.assert_array_equal(np.asarray(out["b"].data), 2 * np.asarray(out["a"].data))


def _gpu_case(rng, H, W, density, coords):
    """Targets carry distinct values (their row-major position + 1), so an allocation names its target."""
    z = np.where(rng.random((H, W)) < density, np.arange(1, H * W + 1).reshape(H, W), 0).astype(np.float32)
    if coords == "int":
        xs, ys = np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64)[::-1].copy()
    elif coords == "aniso":
        xs, ys = np.arange(W) * 30.0, 5000.0 - np.arange(H) * 12.0
    elif coords == "nonuniform":
        xs, ys = np.cumsum(rng.uniform(0.5, 2.0, W)), -np.cumsum(rng.uniform(0.5, 2.0, H))
    else:
        xs, ys = np.linspace(-179.5, 179.5, W), np.linspace(70.0, -70.0, H) if H > 1 else np.array([10.0])
    return z, xs.astype(np.float64), ys.astype(np.float64)


def _check_pick(z, xs, ys, metric, alloc, dirn, br, best):
    """Where targets carry distinct values: the allocated target is one whose key is the brute force's minimum to
    rounding, and the direction is the direction to that target."""
    H, W = z.shape
    pos = {float(v): k for k, v in enumerate(z.ravel()) if v != 0}
    assert np.array_equal(np.isnan(alloc), br < 0)
    m = br >= 0
    k = np.array([pos[float(v)] for v in alloc[m]], np.int64)
    gr, gc = np.full(z.shape, -1), np.full(z.shape, -1)
    gr[m], gc[m] = k // W, k % W
    ii, cc = np.nonzero(m)
    key = _pair_cost(metric, xs, ys, gr[m], gc[m], ii, cc)
    np.testing.assert_allclose(key, best[m], rtol=1e-12, atol=1e-12 * np.abs(best[m]).max(initial=1.0))
    _ulp_close(dirn, _outputs(z, xs, ys, gr, gc, metric, 2))


SHAPES = [(1, 1), (1, 300), (300, 1), (257, 1031), (133, 77), (700, 45)]


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [0, 2, 1])
def test_gpu_equals_the_brute_force(metric):
    rng = np.random.default_rng(7 + metric)
    for H, W in SHAPES:
        for density in (0.0, 1e-4, 0.02, 0.5, 1.0):
            for coords in (["int", "aniso", "nonuniform"] if metric != 1 else ["lonlat"]):
                z, xs, ys = _gpu_case(rng, H, W, density, coords)
                if density == 1e-4:
                    i, j = rng.integers(H), rng.integers(W)
                    z[i, j] = i * W + j + 1
                if H * W * max(1, np.count_nonzero(z)) > 3e7:
                    continue   # the brute force would take minutes; the at-scale test covers large rasters
                br, bc, best = _brute((z != 0) & np.isfinite(z), xs, ys, metric)
                exact = coords in ("int", "aniso") and metric != 1
                d = _run(z, xs, ys, metric, 0)
                _ulp_close(d, _outputs(z, xs, ys, br, bc, metric, 0))
                got = {mode: _run(z, xs, ys, metric, mode) for mode in (1, 2)}
                if exact:
                    for mode in (1, 2):
                        want = _outputs(z, xs, ys, br, bc, metric, mode)
                        assert np.array_equal(got[mode], want, equal_nan=True), (H, W, density, coords, mode)
                    continue
                _check_pick(z, xs, ys, metric, got[1], got[2], br, best)


@pytest.mark.gpu
def test_gpu_targets_nan_inf_and_max_distance():
    rng = np.random.default_rng(11)
    z = rng.integers(0, 5, (60, 70)).astype(np.float32)
    z[rng.random(z.shape) < 0.05] = np.nan
    z[rng.random(z.shape) < 0.02] = np.inf
    z[rng.random(z.shape) < 0.02] = -np.inf
    z[5, 5] = np.float32(0.1)
    xs, ys = np.arange(70.0), np.arange(60.0)
    for tv in ([], [3], [np.inf, 2], [0.1], [np.float32(0.1)], [np.nan], [1, np.nan, 4]):
        vals = np.asarray(tv)
        mask = np.isin(z.astype(np.float64), vals.astype(np.float64)) if vals.size else (z != 0) & np.isfinite(z)
        br, bc, _ = _brute(mask, xs, ys, 0)
        for mode in (0, 1, 2):
            for md in (np.inf, 3.0, 2.0 ** 0.5):   # targets exactly at the limit are kept
                got = _run(z, xs, ys, 0, mode, tv, md)
                assert np.array_equal(got, _outputs(z, xs, ys, br, bc, 0, mode, md), equal_nan=True), (tv, mode, md)
    assert np.isnan(_run(z, xs, ys, 0, 0, [np.nan])).all()


@pytest.mark.gpu
def test_gpu_cell_types():
    rng = np.random.default_rng(12)
    base = rng.integers(0, 4, (50, 61))
    xs, ys = np.arange(61.0), np.arange(50.0)
    want = _run(base.astype(np.float32), xs, ys, 0, 1)
    for dt in (np.float64, np.int32, np.int64, np.int16, np.uint16, np.int8, np.uint8, np.uint32, np.float16):
        assert np.array_equal(_run(base.astype(dt), xs, ys, 0, 1), want, equal_nan=True), dt


@pytest.mark.gpu
def test_gpu_against_the_reference_outputs(golden):
    names = sorted({k.split("_")[1] for k in golden if k.startswith("case_") and k.endswith("_data")})
    for name in names:
        z, xs, ys = golden["case_%s_data" % name], golden["case_%s_x" % name], golden["case_%s_y" % name]
        mask = (z != 0) & np.isfinite(z)
        for mname, metric in METRICS.items():
            key = "case_%s_%s_" % (name, mname)
            if key + "proximity" not in golden:
                continue
            ref = golden[key + "proximity"]
            got = _run(z, xs, ys, metric, 0)
            assert np.array_equal(np.isnan(got), np.isnan(ref))
            m = ~np.isnan(ref)
            tol = np.spacing(np.abs(ref[m]).astype(np.float32))
            assert (got[m] <= ref[m] + tol).all(), (name, mname)
            br, bc, best = _brute(mask, xs, ys, metric)
            bd = _outputs(z, xs, ys, br, bc, metric, 0)
            differ = np.abs(got - ref) > np.spacing(np.abs(ref).astype(np.float32))
            assert (bd[differ] < ref[differ]).all(), (name, mname)
            # allocation and direction where the nearest target is unique and the reference found it
            ti, tc = np.nonzero(mask)
            ii, cc = np.nonzero(m & ~differ)
            cost = _pair_cost(metric, xs, ys, ti[None, :], tc[None, :], ii[:, None], cc[:, None])
            srt = np.sort(cost, axis=1)
            uniq = (srt[:, 1] - srt[:, 0] > 1e-9 * np.abs(srt[:, 0]).clip(1e-12)) if srt.shape[1] > 1 else \
                np.ones(ii.size, bool)
            for mode, mn in ((1, "allocation"), (2, "direction")):
                g = _run(z, xs, ys, metric, mode)[ii[uniq], cc[uniq]]
                r = golden[key + mn][ii[uniq], cc[uniq]]
                np.testing.assert_allclose(g, r, rtol=1e-5, atol=1e-4 if mode == 2 else 0)


@pytest.mark.gpu
def test_gpu_band_split_does_not_change_the_output():
    """Bit-identical output for every band split, and across two identical calls."""
    rng = np.random.default_rng(13)
    for metric, coords in ((0, "int"), (0, "nonuniform"), (2, "aniso"), (2, "nonuniform"), (1, "lonlat")):
        for H, W, density in ((1000, 300, 0.003), (700, 2100, 0.0005)):
            z, xs, ys = _gpu_case(rng, H, W, density, coords)
            for mode in (0, 1, 2):
                ref = _run(z, xs, ys, metric, mode)
                for br in (H, 500, 143, 64, 7, 0, 0):
                    got = _run(z, xs, ys, metric, mode, band_rows=br)
                    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), (metric, coords, mode, br)


@pytest.mark.gpu
def test_gpu_great_circle_wraps_in_every_warp_of_a_wide_row():
    """Rows 4096 cells wide (16 tiles of 8 warps in the row pass) whose nearest target for the eastern cells is
    the row's first, across the antimeridian; and a raster whose coordinates hold both -180 and 180, where every
    target must stay its own nearest target."""
    W = 4096
    xs = np.linspace(-179.95, 179.95, W)
    ys = np.array([-40.0, -10.0, 0.0, 25.0, 60.0])
    z = np.zeros((5, W), np.float32)
    for i, j in enumerate((0, 1, 3, 0, 2)):
        z[i, j] = 10 + i                  # the row's first target, just east of -180
        z[i, 900 + 37 * i] = 20 + i       # a second one, far from the eastern cells
    mask = z != 0
    br, bc, best = _brute(mask, xs, ys, 1)
    assert (bc[:, 3000:] <= 3).all()      # the eastern cells take a first target, across the antimeridian
    _ulp_close(_run(z, xs, ys, 1, 0), _outputs(z, xs, ys, br, bc, 1, 0))
    # cell (0, 450) lies halfway between its row's two targets: either is right
    _check_pick(z, xs, ys, 1, _run(z, xs, ys, 1, 1), _run(z, xs, ys, 1, 2), br, best)
    xs2 = np.linspace(-180.0, 180.0, 361)
    ys2 = np.linspace(-60.0, 60.0, 7)
    z2 = np.zeros((7, 361), np.float32)
    z2[:, 0], z2[:, 360], z2[3, 100] = 1.0, 2.0, 3.0
    assert (_run(z2, xs2, ys2, 1, 0)[z2 != 0] == 0).all()
    assert np.array_equal(_run(z2, xs2, ys2, 1, 1)[z2 != 0], z2[z2 != 0])
    assert (_run(z2, xs2, ys2, 1, 2)[z2 != 0] == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(8192, 8192), (16384, 4096)])
def test_gpu_at_scale_against_scipy(shape):
    ndimage = pytest.importorskip("scipy.ndimage")
    rng = np.random.default_rng(14)
    H, W = shape
    z = np.zeros(shape, np.float32)
    n = 4000
    z[rng.integers(0, H, n), rng.integers(0, W, n)] = rng.integers(1, 1000, n).astype(np.float32)
    xs, ys = np.arange(W) * 1.0, np.arange(H)[::-1] * 1.0
    d = _run(z, xs, ys, 0, 0)
    edt = ndimage.distance_transform_edt(z == 0, sampling=(1.0, 1.0))
    want = np.sqrt((edt.astype(np.float32) ** 2).astype(np.float64)).astype(np.float32)
    assert (np.abs(d - want) <= np.spacing(want)).all()
    a = _run(z, xs, ys, 0, 1)
    # every allocated value belongs to a target at the minimum distance
    sub = (slice(0, H, 97), slice(0, W, 89))
    ii, cc = np.meshgrid(np.arange(H)[sub[0]], np.arange(W)[sub[1]], indexing="ij")
    ti, tc = np.nonzero(z)
    cost = (tc[None, :] - cc.ravel()[:, None]) ** 2.0 + (ti[None, :] - ii.ravel()[:, None]) ** 2.0
    ok = (cost == cost.min(axis=1, keepdims=True)) & (z[ti, tc][None, :] == a[sub].ravel()[:, None])
    assert ok.any(axis=1).all()

"""classify on the GPU: every golden case of the reference (bit for bit for the seven exact schemes, within the
stated tolerance for std_mean and head_tail_breaks), the device order statistics, sort and moments against
NumPy, every cell type, containers, views, ragged and > 2^31-cell rasters, metadata and Datasets."""
import json
import os

import numpy as np
import pytest

import xrspatial_b200 as xb
from xrspatial_b200 import classify as cl

torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
EXACT = {"binary", "reclassify", "quantile", "percentiles", "box_plot", "equal_interval", "maximum_breaks"}
TOL = 2.0 ** -20      # std_mean / head_tail_breaks: breaks within TOL * max|finite value| (DESIGN.md section 4.11)
BINS = {"quantile": lambda r, kw: cl.quantile_bins(r, kw["k"]),
        "percentiles": lambda r, kw: cl.percentiles_bins(r, kw.get("pct", [1, 10, 50, 90, 99])),
        "box_plot": lambda r, kw: cl.box_plot_bins(r, kw.get("hinge", 1.5)),
        "equal_interval": lambda r, kw: cl.equal_interval_bins(r, kw.get("k", 5))[0],
        "std_mean": lambda r, kw: cl.std_mean_bins(r),
        "head_tail_breaks": lambda r, kw: cl.head_tail_bins(r),
        "maximum_breaks": lambda r, kw: cl.maximum_breaks_bins(r.max_break_stats(), kw.get("k", 5))}

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(GOLDEN, "classify_reference.npz"), allow_pickle=False))


def golden_calls(g):
    for case, fn, kw, tag in json.loads(str(g["calls"])):
        kw = {k: [float(x) if isinstance(x, str) else x for x in v] if isinstance(v, list) else v
              for k, v in kw.items()}
        yield case, fn, kw, tag


def host(x):
    return x.cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def cpu_bin(data, bins, new_values):
    """_cpu_bin for strictly increasing bins: the first bin at or above the cell, NaN past the last."""
    d = np.asarray(data, dtype=np.float64)
    out = np.full(d.shape, np.nan, np.float32)
    nv = np.asarray(new_values).astype(np.float32)
    ok = np.isfinite(d) & (d <= bins[-1])
    out[ok] = nv[np.searchsorted(np.asarray(bins, np.float64), d[ok], side="left")]
    return out


class HostStats:
    def __init__(self, data):
        self.dtype = data.dtype
        self.v = np.sort(data[np.isfinite(data)])

    def finite_count(self):
        return self.v.size

    def order_stats(self, ranks):
        return self.v[np.asarray(ranks)]


def check_near_breaks(got, want, data, bins, scale):
    """Cells may differ only where the value lies within TOL * scale of a break."""
    diff = ~((got == want) | (np.isnan(got) & np.isnan(want)))
    if diff.any():
        v = np.asarray(data, np.float64)[diff]
        dist = np.min(np.abs(v[:, None] - np.asarray(bins)[None, :]), axis=1)
        assert np.all(dist <= TOL * scale)


# ---------------------------------------------------------------------------------------------- golden cases
@pytest.mark.parametrize("container", ["numpy", "torch"])
def test_every_golden_case(golden, container, capsys):
    n = 0
    for case, fn, kw, tag in golden_calls(golden):
        data = golden["case__" + case]
        arr = data.copy() if container == "numpy" else torch.from_numpy(data.copy()).cuda()
        agg = xb.DataArray(arr, dims=("y", "x"))
        if "err__" + tag in golden:
            with pytest.raises(Exception) as e:
                getattr(xb, fn)(agg, **kw)
            assert type(e.value).__name__ == str(golden["err__" + tag]), tag
            continue
        capsys.readouterr()
        res = getattr(xb, fn)(agg, **kw)
        printed = capsys.readouterr().out
        assert printed == (str(golden["stdout__" + tag]) if "stdout__" + tag in golden else ""), tag
        assert isinstance(res.data, np.ndarray if container == "numpy" else torch.Tensor), tag
        got, want = host(res.data), golden["out__" + tag]
        assert got.dtype == want.dtype and got.shape == want.shape, tag
        if "newv__" + tag in golden and golden["newv__" + tag].size < golden["bins__" + tag].size:
            # the reference reads past the end of new_values for the last bins: those cells are NaN here
            b = golden["bins__" + tag]
            x = np.asarray(data, np.float64)
            past = np.isfinite(x) & (x > b[golden["newv__" + tag].size - 1]) & (x <= b[-1])
            assert past.any() and np.isnan(got[past]).all(), tag
            want = np.where(past, np.float32(np.nan), want)
        if fn in BINS:
            bins = BINS[fn](cl._Raster(agg), kw)
            wb = golden["bins__" + tag]
            assert bins.shape == wb.shape, tag
        if fn in EXACT:
            assert np.array_equal(got, want, equal_nan=True), tag
            if fn in BINS:
                assert bins.dtype == wb.dtype and np.array_equal(bins, wb, equal_nan=True), tag
        else:
            fin = data[np.isfinite(data)]
            scale = float(np.abs(fin).max()) if fin.size else 0.0
            assert np.all(np.abs(bins - wb) <= TOL * scale) or np.array_equal(bins, wb, equal_nan=True), tag
            check_near_breaks(got, want, data, wb, scale)
        n += 1
    assert n == sum(1 for *_, tag in golden_calls(golden) if "err__" + tag not in golden)


# ---------------------------------------------------------------------------------------------- device primitives
def test_order_statistics_many_ranks_with_ties_and_non_finite():
    """More distinct prefixes than one histogram launch holds: the batched passes still give every rank."""
    rng = np.random.default_rng(3)
    d = (np.round(rng.normal(0, 300, (1536, 1031)) * 4) / 4).astype(np.float32)
    d[rng.random(d.shape) < 0.02] = np.nan
    d[rng.random(d.shape) < 0.001] = np.inf
    d[rng.random(d.shape) < 0.001] = -np.inf
    d[rng.random(d.shape) < 0.01] = -0.0
    r = cl._Raster(xb.DataArray(torch.from_numpy(d).cuda(), dims=("y", "x")))
    fin = np.sort(d[np.isfinite(d)])
    assert r.finite_count() == fin.size
    ranks = np.unique(np.concatenate([rng.integers(0, fin.size, 700), [0, fin.size - 1]]))
    assert np.array_equal(r.order_stats(ranks), fin[ranks])


@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.int16, np.uint16, np.int32, np.int64])
def test_sort_matches_numpy(dtype):
    rng = np.random.default_rng(7)
    if np.dtype(dtype).kind == "f":
        d = rng.normal(0, 1e3, (517, 389)).astype(dtype)
        d[rng.random(d.shape) < 0.05] = np.nan
    else:
        info = np.iinfo(dtype)
        d = rng.integers(max(info.min, -2**40), min(info.max, 2**40), (517, 389), dtype=dtype)
    r = cl._Raster(xb.DataArray(torch.from_numpy(d).cuda(), dims=("y", "x")))
    keys, n = r.sorted_keys()
    fin = np.sort(d[np.isfinite(d)])
    assert n == fin.size
    got = cl._values(host(keys[:n]).view(cl._key_dtype(np.dtype(dtype))), np.dtype(dtype))
    assert np.array_equal(got, fin)


def test_moments_match_float64_numpy():
    rng = np.random.default_rng(9)
    d = (1e5 + rng.normal(0, 2.0, (2001, 1999))).astype(np.float32)    # a large mean over a small spread
    d[rng.random(d.shape) < 0.03] = np.nan
    d[5, 5] = np.inf
    r = cl._Raster(xb.DataArray(torch.from_numpy(d).cuda(), dims=("y", "x")))
    x = d[np.isfinite(d)].astype(np.float64)
    n, mean, m2, mn, mx = r.moments()
    assert n == x.size and mn == x.min() and mx == x.max()
    assert abs(mean - x.mean()) <= 1e-12 * abs(x.mean())
    assert abs(m2 - ((x - x.mean()) ** 2).sum()) <= 1e-9 * ((x - x.mean()) ** 2).sum()
    t = float(np.float32(1e5 + 1.0))
    n2, mean2 = r.moments(t)[:2]
    assert n2 == (x > t).sum() and abs(mean2 - x[x > t].mean()) <= 1e-12 * mean2
    assert r.moments() == (n, mean, m2, mn, mx)      # the same order of merges every call


# ---------------------------------------------------------------------------------------------- cell types
@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.int16, np.uint16, np.int32, np.int64, np.uint8,
                                   np.int8, np.float16, np.uint32])
def test_cell_types(dtype):
    rng = np.random.default_rng(1)
    d = rng.integers(0, 120, (123, 77)).astype(dtype)
    if np.dtype(dtype).kind == "f":
        d[rng.random(d.shape) < 0.05] = np.nan
    for arr in (d, torch.from_numpy(d).cuda() if dtype != np.uint32 else d):
        agg = xb.DataArray(arr, dims=("y", "x"))
        st = HostStats(d)
        q = cl.quantile_bins(st, 6)
        assert np.array_equal(host(xb.quantile(agg, 6).data), cpu_bin(d, q, np.arange(len(q))), equal_nan=True)
        assert np.array_equal(cl.box_plot_bins(cl._Raster(agg), 1.5), cl.box_plot_bins(st, 1.5))
        b = host(xb.binary(agg, [3, 50, 119.0]).data)
        assert b.dtype == d.dtype
        want = np.where(np.isin(d, [3, 50, 119]), 1, np.where(np.isfinite(d.astype(np.float64)), 0, np.nan))
        assert np.array_equal(b.astype(np.float64), want, equal_nan=True)


# ---------------------------------------------------------------------------------------------- containers and metadata
def test_metadata_name_and_inputs_untouched():
    d = np.arange(30, dtype=np.float32).reshape(5, 6)
    d[0, 0] = np.nan
    coords = {"y": np.arange(5.0), "x": np.arange(6.0) * 2}
    for arr in (d.copy(), torch.from_numpy(d.copy()).cuda()):
        agg = xb.DataArray(arr, dims=("y", "x"), coords=coords, attrs={"res": (2.0, 1.0), "crs": "x"})
        before = host(arr).copy()
        for fn, kw in [("binary", dict(values=[3])), ("reclassify", dict(bins=[10, 20, 30], new_values=[1, 2, 3])),
                       ("quantile", {}), ("percentiles", {}), ("box_plot", {}), ("equal_interval", {}),
                       ("std_mean", {}), ("head_tail_breaks", {}), ("maximum_breaks", {})]:
            res = getattr(xb, fn)(agg, **kw)
            assert res.name == fn and tuple(res.dims) == ("y", "x") and res.attrs == agg.attrs, fn
            assert np.array_equal(np.asarray(res["x"]), coords["x"]), fn
            assert getattr(xb, fn)(agg, name="custom", **kw).name == "custom"
            assert np.array_equal(host(arr), before, equal_nan=True), fn
            if isinstance(arr, torch.Tensor):
                assert isinstance(res.data, torch.Tensor) and res.data.device == arr.device
            else:
                assert isinstance(res.data, np.ndarray)


def test_dataset_input():
    d1 = np.arange(20, dtype=np.float32).reshape(4, 5)
    d2 = d1[::-1].copy() * 3
    ds = xb.Dataset({"a": xb.DataArray(d1, dims=("y", "x")), "b": xb.DataArray(d2, dims=("y", "x"))},
                    attrs={"title": "t"})
    res = xb.quantile(ds, k=3)
    assert set(res.data_vars) == {"a", "b"} and res.attrs == {"title": "t"}
    for v, d in (("a", d1), ("b", d2)):
        assert np.array_equal(res[v].data, xb.quantile(xb.DataArray(d, dims=("y", "x")), k=3).data)


def test_dask_is_not_supported():
    da = pytest.importorskip("dask.array")
    with pytest.raises(NotImplementedError):
        xb.reclassify(xb.DataArray(da.zeros((4, 4)), dims=("y", "x")), [1], [1])


def test_pitched_view_and_ragged_size():
    rng = np.random.default_rng(2)
    big = torch.from_numpy((rng.normal(500, 200, (3001, 3010)) // 0.5 * 0.5).astype(np.float32)).cuda()
    view = big[:, 4:3003]                               # rows 3010 cells apart, 2999 wide
    assert view.stride(0) == 3010 and view.stride(1) == 1
    d = host(view).copy()
    agg = xb.DataArray(view, dims=("y", "x"))
    st = HostStats(d)
    for k in (1, 7, 10):
        q = cl.quantile_bins(st, k)
        assert np.array_equal(cl.quantile_bins(cl._Raster(agg), k), q)
        assert np.array_equal(host(xb.quantile(agg, k).data), cpu_bin(d, q, np.arange(len(q))), equal_nan=True)
    uv = np.unique(d)
    for k in (5, 40):
        idx = np.sort(np.argsort(np.diff(uv), kind="stable")[-(k - 1):])
        want = np.append((uv[idx] + uv[idx + 1]) / 2.0, float(uv[-1]))
        got = cl.maximum_breaks_bins(cl._Raster(agg).max_break_stats(), k)
        assert np.array_equal(got, want)
        assert np.array_equal(host(xb.maximum_breaks(agg, k).data), cpu_bin(d, want, np.arange(k)), equal_nan=True)
    ei, l_cuts = cl.equal_interval_bins(cl._Raster(agg), 5)
    assert np.array_equal(host(xb.equal_interval(agg).data), cpu_bin(d, ei, np.arange(l_cuts)), equal_nan=True)


def test_beyond_2_31_cells():
    H = W = 46341                                        # 2 147 488 281 cells
    need = H * W * 4 * 3 + (4 << 30)
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip("needs %.1f GB of free device memory" % (need / 1e9))
    rows = (torch.arange(H, device="cuda", dtype=torch.int64) * W % 251).to(torch.int32)[:, None]
    x = rows + torch.arange(W, device="cuda", dtype=torch.int32)[None, :]
    x.remainder_(251)
    d = x.to(torch.float32)
    del x
    n = H * W                                           # cell i holds i % 251
    agg = xb.DataArray(d, dims=("y", "x"))
    counts = np.full(251, n // 251) + (np.arange(251) < n % 251)
    csum = np.cumsum(counts)

    class Counted:
        dtype = np.dtype(np.float32)

        def finite_count(self):
            return n

        def order_stats(self, ranks):
            return np.searchsorted(csum, np.asarray(ranks), side="right").astype(np.float32)

    r = cl._Raster(agg)
    assert r.finite_count() == n
    ranks = np.array([0, 1, n // 2, n - 2, n - 1, int(csum[100]), int(csum[100]) - 1])
    assert np.array_equal(r.order_stats(ranks), Counted().order_stats(ranks))
    q = cl.quantile_bins(Counted(), 10)
    assert np.array_equal(cl.quantile_bins(r, 10), q)
    out = xb.reclassify(agg, bins=[100, 200, 250], new_values=[0, 1, 2]).data
    del d, rows
    last = out.view(-1)[-1000:].cpu().numpy()
    idx = np.arange(n - 1000, n) % 251
    assert np.array_equal(last, np.where(idx <= 100, 0, np.where(idx <= 200, 1, 2)).astype(np.float32))
    assert int((out == 0).sum()) == int(csum[100])


# ---------------------------------------------------------------------------------------------- per-cell pass layouts
LAYOUTS = {"64x64": (64, 64, None), "3000x3008": (3000, 3008, None), "3001x2999": (3001, 2999, None),
           "61x77": (61, 77, None), "pitched 130x131 of 160": (130, 131, (160, 8))}


def layout_cells(dtype, layout, rng):
    """(device raster, its host copy) in `layout`: contiguous, or columns 8 .. 138 of a 160-wide raster (rows
    16-byte aligned for every cell type, 131 cells wide: each row ends in a partial vector)."""
    H, W, pitched = LAYOUTS[layout]
    Wb, off = pitched or (W, 0)
    dt = np.dtype(dtype)
    if dt.kind == "f":
        d = (np.round(rng.normal(0, 150, (H, Wb)) * 2) / 2).astype(dt)
        d[rng.random(d.shape) < 0.04] = np.nan
        d[rng.random(d.shape) < 0.01] = np.inf
        d[rng.random(d.shape) < 0.01] = -np.inf
    else:
        lo = 0 if dt.kind == "u" else -300
        d = rng.integers(lo, lo + 601, (H, Wb)).astype(dt)
    t = torch.from_numpy(d).cuda()[:, off:off + W]
    return t, d[:, off:off + W].copy()


@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.int16, np.uint16, np.int32, np.int64])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_per_cell_pass_layouts(dtype, layout):
    """Whole 16-byte vectors, a partial last vector in the same row, and rows whose output is not aligned like
    the input: reclassify and binary against NumPy for every cell type the kernel reads."""
    rng = np.random.default_rng(abs(hash((np.dtype(dtype).str, layout))) % 2**32)
    t, d = layout_cells(dtype, layout, rng)
    if layout.startswith("pitched"):
        assert t.stride(0) * t.element_size() % 16 == 0 and t.data_ptr() % 16 == 0 and t.shape[1] % 2 == 1
    shift = 300 if np.dtype(dtype).kind == "u" else 0
    bins = np.array([-200, -50.5, 0, 10, 120, 250]) + shift
    nv = np.array([1.5, 2, 3, 4, 5, 6.25])
    vals = [-50 + shift, 0 + shift, 7 + shift, 120 + shift, 299 + shift, np.inf, np.nan]
    x = d.astype(np.float64)
    want_b = np.where(np.isin(x, vals), 1.0, np.where(np.isfinite(x), 0.0, np.nan)).astype(dtype)
    for arr in (t, d) if layout == "64x64" else (t,):
        agg = xb.DataArray(arr, dims=("y", "x"))
        got = host(xb.reclassify(agg, bins, nv).data)
        assert got.dtype == np.float32
        assert np.array_equal(got, cpu_bin(d, bins, nv), equal_nan=True)
        b = host(xb.binary(agg, vals).data)
        assert b.dtype == np.dtype(dtype)
        assert np.array_equal(b, want_b, equal_nan=True)


def max_breaks_restated(d, k):
    """classify.py:1191-1202 on the finite cells in their own type."""
    uv = np.unique(d[np.isfinite(d)])
    if len(uv) < k:
        return uv
    diffs = np.diff(uv)
    top = np.sort(np.argsort(diffs, kind="stable")[-min(k - 1, len(diffs)):])
    with np.errstate(over="ignore"):    # int8 sums wrap, as in the reference
        return np.append(np.array([(uv[i] + uv[i + 1]) / 2.0 for i in top]), float(uv[-1]))


@pytest.mark.parametrize("dtype", [np.int8, np.uint8, np.float16])
def test_maximum_breaks_on_widened_cells_takes_gaps_in_their_own_type(dtype):
    """int8 gaps wrap when the range exceeds 127 and float16 gaps round to float16, where the widened type's
    would not."""
    rng = np.random.default_rng(4)
    if dtype == np.float16:
        d = (rng.normal(0, 2000, (257, 263))).astype(np.float16)
        d[rng.random(d.shape) < 0.03] = np.nan
    else:
        info = np.iinfo(dtype)
        d = rng.integers(info.min, int(info.max) + 1, (257, 263)).astype(dtype)
        lo, hi = (-100, 60) if info.min < 0 else (40, 200)
        d[(d > lo) & (d < hi)] = info.min      # a gap of 160: int8's np.diff wraps it to -96
    if dtype == np.int8:
        assert not np.array_equal(max_breaks_restated(d, 5), max_breaks_restated(d.astype(np.int16), 5))
    for arr in (d, torch.from_numpy(d).cuda()):
        agg = xb.DataArray(arr, dims=("y", "x"))
        for k in (2, 5, 9):
            want = max_breaks_restated(d, k)
            got = cl.maximum_breaks_bins(cl._Raster(agg).max_break_stats(), k)
            assert got.dtype == want.dtype and np.array_equal(got, want), k
            assert np.array_equal(host(xb.maximum_breaks(agg, k).data), cpu_bin(d, want, np.arange(len(want))),
                                  equal_nan=True)

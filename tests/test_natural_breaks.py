"""natural_breaks on the GPU: every golden case of the reference bit for bit (breaks, their dtype, every output
cell, the warnings, the exception), the device sample against NumPy's shuffle up to 2^26 cells, the device Jenks
matrices against the NumPy statement of the column passes, cell types, views, Datasets, and a raster of more than
2^31 cells."""
import json
import os
import warnings

import numpy as np
import pytest

import xrspatial_b200 as xb
from xrspatial_b200 import classify as cl
from test_natural_breaks_host import jenks_columns, numpy_sample

torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
ERRORS = {"ValueError": ValueError, "IndexError": IndexError, "TypeError": TypeError,
          "TypingError": TypeError}   # numba's typing error for a non-integer k: TypeError here

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(GOLDEN, "natural_breaks_reference.npz"), allow_pickle=False))


def large_case(seed, h, w):
    """oracle/make_golden_natural_breaks.py's large raster, rebuilt from its seed and shape."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    dem = (300 * np.sin(x / 97.0) * np.cos(y / 131.0) + 0.25 * x).astype(np.float32)
    dem += rng.normal(0, 2, dem.shape).astype(np.float32)
    dem[rng.random(dem.shape) < 0.01] = np.nan
    dem[5, 7] = np.inf
    return dem


def host(x):
    return x.cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def cpu_bin(data, bins, new_values):
    """_cpu_bin for increasing bins: the first bin at or above the cell, NaN past the last."""
    d = np.asarray(data, dtype=np.float64)
    out = np.full(d.shape, np.nan, np.float32)
    nv = np.asarray(new_values).astype(np.float32)
    ok = np.isfinite(d) & (d <= bins[-1])
    pos = np.searchsorted(np.asarray(bins, np.float64), d[ok], side="left")
    out[ok] = np.where(pos < nv.size, nv[np.minimum(pos, nv.size - 1)], np.nan)
    return out


def same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and bool(np.all((a == b) | (np.isnan(a) & np.isnan(b))))


def run(raster, container, kw):
    data = raster if container == "numpy" else torch.as_tensor(raster, device="cuda")
    agg = xb.DataArray(data, dims=("y", "x"))
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        res = xb.natural_breaks(agg, **kw)
    return res, [str(w.message) for w in caught if w.category is Warning]


# ---------------------------------------------------------------------------------------------- golden cases
@pytest.mark.parametrize("container", ["numpy", "torch"])
def test_every_golden_case(golden, container):
    seen = 0
    rasters = {}
    calls = json.loads(str(golden["calls"]))
    for case, kw, tag in calls:
        if case not in rasters:
            rasters[case] = (large_case(*golden["gen__" + case].tolist()) if "gen__" + case in golden
                             else golden["case__" + case])
        raster = rasters[case]
        if "err__" + tag in golden:
            with pytest.raises(ERRORS[str(golden["err__" + tag])]):
                run(raster, container, kw)
            seen += 1
            continue
        r = cl._Raster(xb.DataArray(raster if container == "numpy" else torch.as_tensor(raster, device="cuda")))
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            bins, uvk = cl.natural_breaks_bins(r, kw.get("num_sample", 20000), kw.get("k", 5))
        want = golden["bins__" + tag]
        assert bins.dtype == want.dtype and np.array_equal(bins, want), tag
        assert np.array_equal(np.arange(uvk), golden["newv__" + tag]), tag
        res, msgs = run(raster, container, kw)
        assert msgs == [str(m) for m in golden.get("warn__" + tag, [])], tag
        out = host(res.data)
        assert isinstance(res.data, np.ndarray if container == "numpy" else torch.Tensor)
        assert out.dtype == np.float32 and res.name == kw.get("name", "natural_breaks")
        if want.size == 0:
            # an empty sample (num_sample=0): the reference's _cpu_bin reads past its empty bins array; here no
            # cell has a class
            assert np.isnan(out).all(), tag
        elif "out__" + tag in golden:
            assert same(out, golden["out__" + tag]), tag
        else:
            assert same(out, cpu_bin(raster, want, golden["newv__" + tag])), tag
        seen += 1
    assert seen == len(calls)
    fx = golden["fixture__result_natural_breaks"]
    assert same(host(run(golden["case__ref_elevation"], container, {"k": 5})[0].data), fx)


# ---------------------------------------------------------------------------------------------- the sample
@pytest.mark.parametrize("n", [2, 3, 1000, 2 ** 16, 2 ** 16 + 1, 2 ** 20, 2 ** 20 + 1, 2 ** 24, 2 ** 24 + 1,
                               2 ** 26, 2 ** 26 + 1])
def test_device_sample_is_numpys_shuffle_set(n):
    idx = np.linspace(0, n, n, endpoint=False, dtype=np.uint32)
    np.random.RandomState(cl.NB_SEED).shuffle(idx)
    for s in sorted({1, 8, 20000, n // 3, n - 1}):
        if 1 <= s < n:
            got = cl.sample_indices(n, s, torch.device("cuda")).cpu().numpy()
            assert np.array_equal(got, np.sort(idx[:s]).astype(np.int64)), (n, s)


def test_device_sample_other_seeds():
    for seed in (0, 5489, 2 ** 32 - 1):
        got = cl.sample_indices(300001, 777, torch.device("cuda"), seed).cpu().numpy()
        assert np.array_equal(got, numpy_sample(300001, 777, seed)), seed


def test_more_than_2_to_the_32_cells_raise():
    with pytest.raises(ValueError):
        cl.sample_indices(2 ** 32 + 1, 20000, torch.device("cuda"))


# ---------------------------------------------------------------------------------------------- the Jenks passes
def test_device_jenks_matrices_are_the_column_passes(golden):
    rng = np.random.default_rng(11)
    samples = [(golden["jenks_data__" + t].astype(np.float32), golden["jenks_lcl__" + t].shape[1] - 1, t)
               for t in [k[len("jenks_data__"):] for k in golden if k.startswith("jenks_data__")]]
    samples += [(np.sort(rng.normal(0, 1, 3001).astype(np.float32)), 5, None),
                (np.sort(np.round(rng.gamma(2, 3, 4000)).astype(np.float32)), 3, None),
                (np.sort(rng.normal(5, 1, 1500).astype(np.float32) * 1e4), 9, None),
                (np.array([1.5], np.float32), 4, None), (np.array([1.0, 2.0], np.float32), 2, None)]
    for x, k, tag in samples:
        lcl, var = cl.jenks_matrices(torch.as_tensor(x, device="cuda"), k)
        lcl, var = lcl.cpu().numpy().T, var.cpu().numpy().T
        if tag is not None:
            want_l, want_v = golden["jenks_lcl__" + tag], golden["jenks_var__" + tag]
        else:
            want_l, want_v = jenks_columns(x, k)
        assert np.array_equal(lcl.view(np.uint32), want_l.view(np.uint32)), (x.size, k)
        assert np.array_equal(var.view(np.uint32), want_v.view(np.uint32)), (x.size, k)


# ---------------------------------------------------------------------------------------------- cell types, views
def host_natural_breaks(raster, num_sample, k):
    flat = raster.ravel()
    fin = flat[np.isfinite(flat)] if flat.dtype.kind == "f" else flat
    max_data = float(np.max(fin))
    sample = flat[numpy_sample(flat.size, num_sample)] if num_sample < flat.size else flat
    data = np.sort(sample[np.isfinite(sample)] if sample.dtype.kind == "f" else sample)
    uv = np.unique(data)
    if uv.size < k:
        return uv, uv.size
    lcl = jenks_columns(data.astype(np.float32), k)[0]
    return cl.jenks_backtrack(data, lcl, k, max_data), uv.size


@pytest.mark.parametrize("dtype", ["float32", "float64", "float16", "int8", "uint8", "int16", "uint16", "int32",
                                   "uint32", "int64"])
def test_cell_types(dtype):
    rng = np.random.default_rng(3)
    v = rng.normal(40, 30, (37, 53))
    if np.dtype(dtype).kind == "f":
        raster = v.astype(dtype)
        raster[rng.random(raster.shape) < 0.05] = np.nan
    else:
        info = np.iinfo(dtype)
        raster = np.clip(np.round(v), info.min, info.max).astype(dtype)
    before = raster.copy()
    bins, uvk = host_natural_breaks(raster, 400, 5)
    for container in ("numpy", "torch"):
        res, _ = run(raster, container, dict(num_sample=400, k=5))
        assert same(host(res.data), cpu_bin(raster, bins, np.arange(uvk))), (dtype, container)
    assert np.array_equal(raster, before, equal_nan=True)


def test_pitched_view_and_dataset():
    rng = np.random.default_rng(4)
    base = torch.as_tensor(rng.normal(0, 10, (64, 96)).astype(np.float32), device="cuda")
    view = base[5:60, 7:90]
    keep = base.clone()
    res, _ = run(view, "torch", dict(num_sample=500, k=4))   # run() wraps the tensor as given
    dense = view.contiguous().cpu().numpy()
    bins, uvk = host_natural_breaks(dense, 500, 4)
    assert same(host(res.data), cpu_bin(dense, bins, np.arange(uvk)))
    assert torch.equal(base, keep)
    ds = xb.Dataset({"a": xb.DataArray(dense, dims=("y", "x")), "b": xb.DataArray(dense * 2, dims=("y", "x"))})
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out = xb.natural_breaks(ds, num_sample=500, k=4)
    assert same(out["a"].data, host(res.data))
    bins2, uvk2 = host_natural_breaks(dense * 2, 500, 4)
    assert same(out["b"].data, cpu_bin(dense * 2, bins2, np.arange(uvk2)))


# ---------------------------------------------------------------------------------------------- > 2^31 cells
def test_more_than_2_to_the_31_cells():
    H, W = 32769, 65536      # 2^31 + 2^16 cells of float32
    n = H * W
    t = torch.empty((H, W), dtype=torch.float32, device="cuda")
    t.copy_(torch.arange(W, device="cuda", dtype=torch.float32).remainder_(997).view(1, W))
    t.add_(torch.arange(H, device="cuda", dtype=torch.float32).remainder_(89).view(H, 1))
    a = cl.sample_indices(n, 20000, t.device)
    b = cl.sample_indices(n, 20000, t.device)
    assert torch.equal(a, b)
    ah = a.cpu().numpy()
    assert ah.size == 20000 and ah[0] >= 0 and ah[-1] < n and np.all(np.diff(ah) > 0)
    sample = t.view(-1)[a].cpu().numpy()
    max_data = float(t.max().item())
    data = np.sort(sample)
    uv = np.unique(data)
    lcl = cl.jenks_matrices(torch.as_tensor(data, device="cuda"), 5)[0].cpu().numpy().T
    bins = cl.jenks_backtrack(data, lcl, 5, max_data)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out = xb.natural_breaks(xb.DataArray(t, dims=("y", "x")), k=5).data
    r = cl._Raster(xb.DataArray(t))
    want = r.cells_pass(False, bins, np.arange(uv.size))
    assert torch.equal(torch.nan_to_num(out, nan=-1.0), torch.nan_to_num(want, nan=-1.0))

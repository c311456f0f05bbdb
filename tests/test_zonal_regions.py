"""zonal regions / trim / crop on the GPU: every golden case of the unmodified reference for numpy and torch
inputs, equality with the host build of the rule on large rasters with cross-tile chains, cell types, pitched
views, streams, metadata, and a raster of more than 2^31 cells."""
import numpy as np
import pytest

import xrspatial_b200 as xb
from test_zonal_regions_host import SUFFIX, bounds_cases, build_host, golden, region_cases

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    return build_host(str(tmp_path_factory.mktemp("zrg")))


def _regions(a, n, device=False):
    data = torch.from_numpy(a).cuda() if device else a
    out = xb.regions(xb.DataArray(data, dims=("y", "x")), neighborhood=n).data
    return out.cpu().numpy() if device else out


def _same(got, want):
    assert got.dtype == want.dtype and got.shape == want.shape
    assert np.array_equal(got, want, equal_nan=want.dtype.kind == "f")


def test_every_golden_regions_case_numpy_and_torch():
    g = golden()
    for i, a, n, ref in region_cases(g):
        _same(_regions(a, n), ref)
        _same(_regions(a, n, device=True), ref)


def test_every_golden_bounds_case_numpy_and_torch():
    g = golden()
    for i, a, vals, mode, ref in bounds_cases(g):
        for data in (a, torch.from_numpy(a).cuda()):
            assert xb.zonal._bounds(data, vals, mode, "t") == ref, (i, vals, mode)
            r = xb.DataArray(data, dims=("y", "x"))
            out = xb.crop(r, r, vals) if mode else xb.trim(r, vals)
            t, b, l, rr = ref
            want = a[t:b + 1, l:rr + 1]
            got = out.data.cpu().numpy() if torch.is_tensor(out.data) else out.data
            assert np.array_equal(got, want, equal_nan=True), i


def _serpentine(H, W, gap=2):
    y, x = np.mgrid[0:H, 0:W]
    band = (y // gap) % 4
    return ((band == 0) | ((band == 1) & (x == W - 1)) | (band == 2) | ((band == 3) & (x == 0))).astype(np.float32)


def _ramp(H, W, seed):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W]
    a = 1000.0 + (x + 0.37 * y) * (1e-8 + 1e-5 * 1000.0) * 0.6
    a[rng.random((H, W)) < 0.02] = np.nan
    return a.astype(np.float64)


@pytest.mark.parametrize("case", ["serpentine", "ramp", "random3", "quantised"])
@pytest.mark.parametrize("n", [4, 8])
def test_large_rasters_equal_the_host_build(host, case, n):
    rng = np.random.default_rng(7)
    if case == "serpentine":
        a = _serpentine(4096, 4096)
    elif case == "ramp":
        a = _ramp(2000, 3001, 3)
    elif case == "random3":
        a = rng.integers(0, 3, (1500, 2500)).astype(np.int32)
    else:
        a = np.round(np.cumsum(rng.standard_normal((4096, 4096)).astype(np.float32), axis=1) / 40).astype(np.float32)
    want = host(a, n)
    got = _regions(a, n, device=True)
    _same(got, want)
    _same(_regions(a, n, device=True), got)   # repeated calls give the same labels


@pytest.mark.parametrize("dtype", list(SUFFIX) + ["bool"])
def test_cell_types_streams_and_inputs_unchanged(host, dtype):
    rng = np.random.default_rng(11)
    a = rng.integers(0, 3, (97, 131)).astype(dtype)
    keep = a.copy()
    t = torch.from_numpy(a).cuda()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        out = xb.regions(xb.DataArray(t, dims=("y", "x")), neighborhood=8).data
    s.synchronize()
    got = out.cpu().numpy()
    want = np.ones(a.shape, bool) if dtype == "bool" else host(a, 8)
    if dtype not in ("bool", "float32", "float64"):   # labels past the type's range wrap as a cast of int64
        want = host(a.astype(np.int64), 8).astype(dtype)
    _same(got, want)
    assert np.array_equal(a, keep) and np.array_equal(t.cpu().numpy(), keep)
    tb = xb.zonal._bounds(t, (0,), 1, "crop")
    rows, cols = np.nonzero(a == 0) if dtype != "bool" else np.nonzero(~a)
    assert tb == (rows.min(), rows.max(), cols.min(), cols.max())


def test_pitched_views_and_metadata(host):
    rng = np.random.default_rng(5)
    big = rng.integers(0, 3, (300, 520)).astype(np.float32)
    big[rng.random(big.shape) < 0.05] = np.nan
    view = torch.from_numpy(big).cuda()[7:250, 13:451]
    a = big[7:250, 13:451]
    ys, xs = np.arange(a.shape[0]) * 2.0, np.arange(a.shape[1]) * 3.0
    r = xb.DataArray(view, dims=("y", "x"), coords={"y": ys, "x": xs}, attrs={"res": (3.0, 2.0)}, name="z")
    out = xb.regions(r, neighborhood=4)
    _same(out.data.cpu().numpy(), host(np.ascontiguousarray(a), 4))
    assert out.name == "regions" and out.dims == ("y", "x") and out.attrs == {"res": (3.0, 2.0)}
    z = np.where(np.isnan(a), 0, a)
    z[:20] = 0
    z[:, -9:] = 0
    zr = xb.DataArray(z, dims=("y", "x"), coords={"y": ys, "x": xs}, attrs={"res": (3.0, 2.0)})
    tr = xb.trim(zr, values=(0,))
    assert tr.name == "trim" and tr.attrs == {"res": (3.0, 2.0)}
    rows, cols = np.nonzero(z != 0)
    assert np.array_equal(tr.data, z[rows.min():rows.max() + 1, cols.min():cols.max() + 1])
    assert np.array_equal(np.asarray(tr.coords["y"]), ys[rows.min():rows.max() + 1])
    assert np.array_equal(np.asarray(tr.coords["x"]), xs[cols.min():cols.max() + 1])
    cr = xb.crop(zr, r, zones_ids=(1,))
    rows, cols = np.nonzero(z == 1)
    assert cr.name == "crop"
    assert np.array_equal(cr.data.cpu().numpy(), a[rows.min():rows.max() + 1, cols.min():cols.max() + 1],
                          equal_nan=True)


def test_more_than_2_31_cells():
    H, W = 1 << 16, (1 << 15) + 64   # 2^31 + 2^22 uint8 cells in row stripes: row r is region r + 1
    free, _ = torch.cuda.mem_get_info()
    if free < 48 * 2 ** 30:
        pytest.skip("needs about 45 GB of free device memory")
    rows = (torch.arange(H, device="cuda") % 2).to(torch.uint8)
    t = rows[:, None].expand(H, W).contiguous()
    del rows
    out = xb.regions(xb.DataArray(t, dims=("y", "x")), neighborhood=4).data
    want = ((torch.arange(H, device="cuda") + 1) % 256).to(torch.uint8)
    assert torch.equal(out[:, 0], want) and torch.equal(out[:, -1], want)
    assert bool((out == want[:, None]).all())
    del out
    assert xb.zonal._bounds(t, (1,), 1, "crop") == (1, H - 1, 0, W - 1)

"""GPU parity: the CUDA path (called through the C ABI by the public API) vs the pinned CPU
oracle and vs the committed reference outputs.  Runs on an H100 (`-m gpu`)."""
import numpy as np
import pytest

import oracle as o
from helpers import assert_aspect_close, assert_close_f32, terrain
from test_geodesic_edges import check, expect

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

DEMS = ["smooth", "water", "nans", "integer", "rough", "tiny", "rand_2x4", "rand_10x15"]
STATS = ["mean", "max", "min", "range", "std", "var", "sum"]


@pytest.fixture(scope="module")
def xb():
    import xrspatial_b200
    assert torch.cuda.is_available(), "these tests need a CUDA device"
    return xrspatial_b200


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def da(xb, data, res=(30.0, 30.0), name="r"):
    return xb.DataArray(data, dims=("y", "x"), attrs={"res": res}, name=name)


def host(x):
    d = x.data
    return d.cpu().numpy() if hasattr(d, "cpu") else np.asarray(d)


def used_tma(xb):
    return xb._lib.lib().xrs_debug_last_used_tma()


# ----------------------------------------------------------------- committed reference outputs
@pytest.mark.parametrize("case", DEMS)
def test_surface_vs_reference_outputs(xb, refout, case):
    z = refout["dem." + case]
    agg = da(xb, dev(z))
    assert_close_f32(host(xb.slope(agg)), refout["slope." + case], what="slope " + case)
    assert_close_f32(host(xb.slope(da(xb, dev(z), res=(10.0, 25.5)))), refout["slope_aniso." + case],
                     what="slope aniso " + case)
    assert_aspect_close(host(xb.aspect(agg)), refout["aspect." + case], what=case)
    ref = refout["curvature." + case]
    assert_close_f32(host(xb.curvature(agg)), ref, atol=1e-6 * max(1.0, np.nanmax(np.abs(ref)) if np.isfinite(ref).any() else 1.0),
                     what="curvature " + case)
    assert_close_f32(host(xb.hillshade(agg)), refout["hillshade." + case], what="hillshade " + case)
    assert_close_f32(host(xb.hillshade(agg, azimuth=315, angle_altitude=45)),
                     refout["hillshade_az315_alt45." + case], what="hillshade2 " + case)


@pytest.mark.parametrize("case", DEMS)
def test_focal_mean_vs_reference_outputs(xb, refout, case):
    z = refout["dem." + case]
    # device f32 path (values = oracle rounded to f32), device f64 path (1e-12), host path (f64)
    assert_close_f32(host(xb.mean(da(xb, dev(z)))), refout["focal_mean." + case], atol=0, what="mean f32")
    out64 = host(xb.mean(da(xb, dev(z.astype(np.float64)))))
    assert out64.dtype == np.float64
    np.testing.assert_allclose(out64, refout["focal_mean." + case], rtol=1e-12, atol=0, equal_nan=True)
    out3 = host(xb.mean(da(xb, dev(z.astype(np.float64))), passes=3))
    np.testing.assert_allclose(out3, refout["focal_mean_p3." + case], rtol=1e-12, atol=0, equal_nan=True)
    oute = host(xb.mean(da(xb, dev(z.astype(np.float64))), excludes=[np.nan, 0.0]))
    np.testing.assert_allclose(oute, refout["focal_mean_ex." + case], rtol=1e-12, atol=0, equal_nan=True)
    outh = xb.mean(da(xb, z)).data  # numpy in -> numpy float64 out
    assert isinstance(outh, np.ndarray) and outh.dtype == np.float64
    np.testing.assert_allclose(outh, refout["focal_mean." + case], rtol=1e-12, atol=0, equal_nan=True)


@pytest.mark.parametrize("kn", ["box3", "box9", "mixed5", "mixed3x7", "mixed25", "int3"])
def test_convolve_vs_reference_outputs(xb, refout, kn):
    from xrspatial_b200.convolution import convolve_2d
    k = refout["conv.kernel." + kn]
    for key, okey in (("conv.dem", "conv.out." + kn), ("conv.dem_nan", "conv.out_nan." + kn)):
        ref = refout[okey]
        scale = np.nanmax(np.abs(ref[np.isfinite(ref)])) if np.isfinite(ref).any() else 1.0
        got = convolve_2d(dev(refout[key]), k).cpu().numpy()
        assert_close_f32(got, ref, atol=1e-6 * scale, what="conv " + kn)


@pytest.mark.parametrize("mn", ["circle3", "full3", "annulus5", "rect3x5", "weights3"])
def test_focal_stats_vs_reference_outputs(xb, refout, mn):
    from xrspatial_b200 import focal
    agg = da(xb, dev(refout["apply.dem"]))
    res = focal.focal_stats(agg, refout["apply.mask." + mn], stats_funcs=STATS)
    assert res.dims[0] == "stats" and tuple(res.shape) == (7,) + refout["apply.dem"].shape
    got = host(res)
    for i, s in enumerate(STATS):
        ref = refout["apply.out.%s.%s" % (mn, s)]
        atol = 1e-6 * np.nanmax(np.abs(ref)) if s in ("var",) else 1e-6
        assert_close_f32(got[i], ref, atol=atol, what="%s %s" % (mn, s))


def test_multispectral_vs_reference_outputs(xb, refout):
    r = refout
    b = {k: da(xb, dev(r["ms." + k])) for k in ("nir", "red", "blue", "green", "swir", "tir")}
    eq = lambda got, key: np.testing.assert_array_equal(host(got), r[key], err_msg=key)  # noqa: E731
    eq(xb.ndvi(b["nir"], b["red"]), "ms.ndvi")
    eq(xb.savi(b["nir"], b["red"]), "ms.savi")
    eq(xb.savi(b["nir"], b["red"], soil_factor=0.5), "ms.savi_L05")
    eq(xb.evi(b["nir"], b["red"], b["blue"]), "ms.evi")
    eq(xb.arvi(b["nir"], b["red"], b["blue"]), "ms.arvi")
    eq(xb.gci(b["nir"], b["green"]), "ms.gci")
    eq(xb.sipi(b["nir"], b["red"], b["blue"]), "ms.sipi")
    eq(xb.ebbi(b["red"], b["swir"], b["tir"]), "ms.ebbi")
    # host (numpy) path returns numpy
    out = xb.ndvi(da(xb, r["ms.nir"]), da(xb, r["ms.red"])).data
    assert isinstance(out, np.ndarray)
    np.testing.assert_array_equal(out, r["ms.ndvi"])


def check_zonal(df, ref, prefix, cols, rtol):
    np.testing.assert_array_equal(np.asarray(df["zone"], dtype=np.float64), ref[prefix + "zone"].astype(np.float64))
    for c in cols:
        got, exp = np.asarray(df[c], dtype=np.float64), ref[prefix + c]
        if c in ("count", "min", "max"):
            np.testing.assert_array_equal(got, exp, err_msg=c)  # bit-exact
        else:
            np.testing.assert_allclose(got, exp, rtol=rtol, atol=rtol * np.nanmax(np.abs(exp)), equal_nan=True,
                                       err_msg=c)


def test_zonal_vs_reference_outputs(xb, refout):
    r = refout
    cols = ["mean", "max", "min", "sum", "std", "var", "count"]
    zones, values = da(xb, dev(r["zonal.zones_i32"])), da(xb, dev(r["zonal.values_f32"]))
    df = xb.zonal_stats(zones, values)
    check_zonal(df, r, "zonal.f32_i32.", cols, 1e-5)
    df = xb.zonal_stats(zones, values, zone_ids=[3, 7, 100, 999], nodata_values=0.0)
    check_zonal(df, r, "zonal.f32_i32_ids_nodata.", cols, 1e-5)
    df = xb.zonal_stats(da(xb, dev(r["zonal.zones_f64"])), da(xb, dev(r["zonal.values_f64"])))
    check_zonal(df, r, "zonal.f64_f64.", cols, 1e-12)
    arr = xb.zonal_stats(zones, values, zone_ids=[3, 7], stats_funcs=["mean", "count"],
                         return_type="xarray.DataArray")
    np.testing.assert_allclose(host(arr), r["zonal.f32_i32.broadcast_mean_count_3_7"], rtol=1e-5, equal_nan=True)
    # host path
    dfh = xb.zonal_stats(da(xb, r["zonal.zones_i32"]), da(xb, r["zonal.values_f32"]))
    check_zonal(dfh, r, "zonal.f32_i32.", cols, 1e-5)
    assert dfh["zone"].dtype == np.int32


# ----------------------------------------------------------------- TMA path vs the oracle
@pytest.mark.parametrize("shape,kw", [((300, 512), {}), ((517, 1024), dict(nans=0.01)),
                                      ((1030, 260), dict(water=True)), ((64, 128), {}),
                                      ((2048, 2048), {})])
def test_tma_path_vs_oracle(xb, shape, kw):
    rng = np.random.default_rng(hash(shape) % 1000)
    z = terrain(rng, *shape, **kw)
    agg = da(xb, dev(z))
    s = host(xb.slope(agg))
    assert used_tma(xb) == 1
    assert_close_f32(s, o.slope(z, 30.0, 30.0, nthreads=8), what="slope")
    assert_aspect_close(host(xb.aspect(agg)), o.aspect(z, nthreads=8))
    ref = o.curvature(z, 30.0, nthreads=8)
    assert_close_f32(host(xb.curvature(agg)), ref, atol=1e-6 * np.nanmax(np.abs(ref)), what="curvature")
    assert_close_f32(host(xb.hillshade(agg)), o.hillshade(z, nthreads=8), what="hillshade")
    assert_close_f32(host(xb.mean(agg)), o.focal_mean(z, nthreads=8), atol=0, what="focal mean")
    assert used_tma(xb) == 1
    out64 = host(xb.mean(da(xb, dev(z.astype(np.float64))), passes=2))
    np.testing.assert_allclose(out64, o.focal_mean(z, passes=2, nthreads=8), rtol=1e-12, equal_nan=True)
    # fused suite == individual kernels, bit for bit
    suite = xb.surface_suite(agg)
    np.testing.assert_array_equal(host(suite["slope"]), s)
    np.testing.assert_array_equal(host(suite["aspect"]), host(xb.aspect(agg)))
    np.testing.assert_array_equal(host(suite["curvature"]), host(xb.curvature(agg)))
    np.testing.assert_array_equal(host(suite["hillshade"]), host(xb.hillshade(agg)))


def test_tma_and_direct_kernels_agree_bitwise(xb):
    """Same operator code behind both loaders: a W%4==0 raster (TMA) and the same raster seen
    through a 1-column-shifted, non-16-byte-aligned view (direct loads) give identical cells."""
    rng = np.random.default_rng(5)
    z = terrain(rng, 200, 257, nans=0.02)
    big = dev(z)
    view = big[:, 1:]               # 256 wide, base pointer offset by 4 bytes -> direct kernel
    a = xb.slope(da(xb, view))
    assert used_tma(xb) == 0
    b = xb.slope(da(xb, view.contiguous()))
    assert used_tma(xb) == 1
    np.testing.assert_array_equal(host(a), host(b))


def test_host_path_matches_device_path(xb):
    rng = np.random.default_rng(11)
    z = terrain(rng, 700, 640, nans=0.01)
    for fn in (xb.slope, xb.aspect, xb.curvature, xb.hillshade):
        h = fn(da(xb, z)).data
        d = fn(da(xb, dev(z))).data
        assert isinstance(h, np.ndarray) and h.dtype == np.float32
        np.testing.assert_array_equal(h, d.cpu().numpy(), err_msg=fn.__name__)
    assert not np.shares_memory(z, h)


def test_host_path_chunked_rows_invariant(xb):
    """The host engine stripes rows in chunks with halos; force many chunks with a wide raster
    and check against the oracle (partition invariance, SURVEY.md 8e)."""
    rng = np.random.default_rng(12)
    z = terrain(rng, 300, 32768 * 2)
    out = xb.slope(da(xb, z)).data      # 256 KiB rows -> 128 rows per chunk -> 3 chunks
    assert_close_f32(out, o.slope(z, 30.0, 30.0, nthreads=8), what="chunked slope")
    from xrspatial_b200.convolution import convolve_2d
    k = np.ones((9, 9)) / 81.0
    got = convolve_2d(z[:, :4096].copy(), k)
    ref = o.convolve_2d(z[:, :4096], k, nthreads=8)
    assert_close_f32(got, ref, atol=1e-6 * np.nanmax(np.abs(ref)), what="host convolve")


@pytest.mark.parametrize("k", [3, 5, 7, 9, 11, 13, 15, 25])
def test_convolve_sizes_vs_oracle(xb, k):
    from xrspatial_b200.convolution import convolve_2d
    rng = np.random.default_rng(k)
    z = terrain(rng, 260, 384, nans=0.001)
    for kern in (np.ones((k, k)) / (k * k), rng.standard_normal((k, k))):
        ref = o.convolve_2d(z, kern, nthreads=8)
        got = convolve_2d(dev(z), kern).cpu().numpy()
        assert_close_f32(got, ref, atol=1e-6 * np.nanmax(np.abs(ref[np.isfinite(ref)])), what="conv k=%d" % k)


@pytest.mark.parametrize("kh,kw", [(5, 5), (9, 9), (25, 25), (3, 7), (7, 3), (1, 5), (25, 3)])
def test_convolve_uniform_kernels_take_the_box_path(xb, kh, kw):
    """All-equal taps (np.ones / k**2, the mean filter) go through the running-box kernel; NaN / inf cells are
    kept out of the running sums: NaN windows are NaN, inf windows come back through the tap-by-tap recompute."""
    from xrspatial_b200.convolution import convolve_2d
    rng = np.random.default_rng(100 * kh + kw)
    z = terrain(rng, 150, 388)
    dirty = z.copy()
    dirty[20, 30] = np.nan
    dirty[70, 200] = np.inf
    dirty[100, 300] = -np.inf
    dirty[149, 387] = np.nan
    for w in (1.0 / (kh * kw), -0.37, 0.0):
        kern = np.full((kh, kw), w)
        for data in (z, dirty, (z + 1e6).astype(np.float32)):
            ref = o.convolve_2d(data, kern, nthreads=8)
            got = convolve_2d(dev(data), kern).cpu().numpy()
            assert used_tma(xb) == 3
            fin = np.isfinite(ref)
            scale = np.abs(ref[fin]).max() if fin.any() else 1.0
            assert_close_f32(got, ref, atol=1e-6 * max(scale, 1e-30), what="box %dx%d w=%g" % (kh, kw, w))
    # one tap off by an ulp: generic tiled kernel
    kern = np.full((kh, kw), 0.25)
    kern[0, 0] = np.nextafter(0.25, 1.0)
    if (kh, kw) != (3, 3):
        convolve_2d(dev(z), kern)
        assert used_tma(xb) == 4


def test_convolve_box_path_small_and_ragged_rasters(xb):
    from xrspatial_b200.convolution import convolve_2d
    rng = np.random.default_rng(77)
    kern = np.ones((9, 9)) / 81.0
    for h, w in ((5, 8), (9, 12), (33, 128), (64, 132), (70, 260)):
        z = terrain(rng, h, w)
        ref = o.convolve_2d(z, kern, nthreads=4)
        got = convolve_2d(dev(z), kern).cpu().numpy()
        assert used_tma(xb) == 3
        assert_close_f32(got, ref, atol=1e-6 * 4000.0, what="box 9x9 on %dx%d" % (h, w))
    z = terrain(rng, 40, 131)            # W % 4 != 0: bounds-checked fallback
    got = convolve_2d(dev(z), kern).cpu().numpy()
    assert used_tma(xb) == 5
    assert_close_f32(got, o.convolve_2d(z, kern, nthreads=4), atol=1e-6 * 4000.0, what="box 9x9 ragged")


def test_focal_stats_multi_abi_ragged_width_falls_back_per_plane(xb):
    """xrs_focal_stats_multi_f32 called directly on a raster TMA cannot describe (W % 4 != 0): the C
    side serves it plane by plane with the bounds-checked kernel; same values as the oracle."""
    import ctypes
    from xrspatial_b200 import _lib
    rng = np.random.default_rng(5)
    z = terrain(rng, 37, 131, nans=0.02)
    t = dev(z)
    kern = np.ones((3, 3))
    names = ["sum", "mean", "max"]
    ids = (ctypes.c_int * 3)(*[_lib.STATS[n] for n in names])
    # plane stride must be a 16-byte multiple covering one plane: use a padded buffer
    stride = (37 * 131 * 4 + 15) // 16 * 16
    buf = torch.empty(3 * stride // 4, dtype=torch.float32, device="cuda")
    _lib.call("xrs_focal_stats_multi_f32", ctypes.c_void_p(t.data_ptr()), 131 * 4, ctypes.c_void_p(buf.data_ptr()),
              131 * 4, stride, 37, 131, kern.ctypes.data_as(ctypes.c_void_p), 3, 3, ids, 3,
              ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    assert used_tma(xb) == 8          # the bounds-checked single-statistic kernel served every plane
    for i, n in enumerate(names):
        got = buf[i * stride // 4: i * stride // 4 + 37 * 131].reshape(37, 131).cpu().numpy()
        assert_close_f32(got, o.focal_apply(z, kern, n, nthreads=4), what="multi fallback " + n)
    with pytest.raises(ValueError):
        _lib.call("xrs_focal_stats_multi_f32", ctypes.c_void_p(t.data_ptr()), 131 * 4, ctypes.c_void_p(buf.data_ptr()),
                  131 * 4, stride, 37, 131, kern.ctypes.data_as(ctypes.c_void_p), 3, 3,
                  (ctypes.c_int * 2)(0, 0), 2, None)            # a statistic requested twice


def test_focal_stats_tma_vs_oracle(xb):
    from xrspatial_b200 import focal
    from xrspatial_b200.convolution import circle_kernel
    rng = np.random.default_rng(3)
    z = terrain(rng, 130, 256, nans=0.03)
    kern = circle_kernel(1, 1, 3)
    res = host(focal.focal_stats(da(xb, dev(z)), kern, stats_funcs=STATS))
    assert used_tma(xb) == 6          # all seven statistics from the fused one-pass kernel
    for i, s in enumerate(STATS):
        ref = o.focal_apply(z, kern, s, nthreads=8)
        atol = 1e-6 * np.nanmax(np.abs(ref)) if s == "var" else 1e-6
        assert_close_f32(res[i], ref, atol=atol, what=s)


@pytest.mark.parametrize("stats", [["mean", "max", "min", "range", "std", "var", "sum"], ["sum", "std"],
                                   ["range", "mean"], ["var", "min", "max"]])
def test_focal_stats_fused_equals_per_statistic_apply(xb, stats):
    """The fused kernel must give, plane by plane, exactly what one `apply` per statistic gives."""
    from xrspatial_b200 import focal
    from xrspatial_b200.convolution import annulus_kernel, circle_kernel
    rng = np.random.default_rng(11)
    z = terrain(rng, 150, 388, nans=0.05)
    z[40:60, 100:140] = np.nan          # a window-sized hole: all-NaN windows
    agg = da(xb, dev(z))
    for kern in (circle_kernel(1, 1, 2), annulus_kernel(1, 1, 3, 1), np.ones((3, 5))):
        fused = focal.focal_stats(agg, kern, stats_funcs=stats)
        assert used_tma(xb) == 6
        assert fused.dims == ("stats", "y", "x") and list(fused.coords["stats"]) == stats
        got = host(fused)
        for i, s in enumerate(stats):
            one = host(focal.apply(agg, kern, func=s))
            np.testing.assert_array_equal(got[i], one, err_msg="%s plane differs from apply" % s)
            ref = o.focal_apply(z, kern, s, nthreads=8)
            atol = 1e-6 * np.nanmax(np.abs(ref)) if s == "var" else 1e-6
            assert_close_f32(got[i], ref, atol=atol, what=s)


@pytest.mark.parametrize("stats", [["mean"], ["var"], ["sum", "min", "max"], STATS])
def test_focal_stats_one_call_on_any_width(xb, stats, monkeypatch):
    """On a device raster whose width is not a multiple of 4, and for a single statistic, focal_stats makes
    one xrs_focal_stats_multi_f32 call and returns what stacking one `apply` per statistic returns."""
    import pandas as pd
    from xrspatial_b200 import _lib, focal
    from xrspatial_b200._xr import concat
    from xrspatial_b200.convolution import circle_kernel
    rng = np.random.default_rng(17)
    z = terrain(rng, 37, 131, nans=0.05)
    agg = xb.DataArray(dev(z), dims=("y", "x"), coords={"y": np.arange(37)[::-1], "x": np.arange(131) * 2.0},
                       attrs={"res": (1, 1), "crs": "x"}, name="dem")
    real_call = _lib.call
    for kern in (circle_kernel(1, 1, 2), np.ones((3, 3))):
        want = concat([focal.apply(agg, kern, func=s) for s in stats], pd.Index(stats, name="stats", dtype=object))
        calls = []
        monkeypatch.setattr(_lib, "call", lambda name, *a: (calls.append(name), real_call(name, *a))[1])
        got = focal.focal_stats(agg, kern, stats_funcs=stats)
        monkeypatch.setattr(_lib, "call", real_call)
        assert calls == ["xrs_focal_stats_multi_f32"]
        assert got.dims == want.dims and got.name == want.name and got.attrs == want.attrs
        assert list(got.coords) == list(want.coords)
        for c in want.coords:
            np.testing.assert_array_equal(np.asarray(got.coords[c]), np.asarray(want.coords[c]))
        assert got.data.dtype == want.data.dtype and tuple(got.shape) == tuple(want.shape)
        np.testing.assert_array_equal(host(got), host(want))


def test_input_not_modified_and_metadata(xb):
    rng = np.random.default_rng(1)
    z = terrain(rng, 40, 64)
    t = dev(z)
    agg = xb.DataArray(t, dims=("y", "x"), coords={"y": np.arange(40)[::-1], "x": np.arange(64)},
                       attrs={"res": (1, 1), "crs": "x"}, name="dem")
    out = xb.slope(agg, name="myslope")
    assert out.name == "myslope" and out.dims == agg.dims and out.attrs == agg.attrs
    assert type(out.data) is type(t) and tuple(out.shape) == z.shape and out.data.dtype == torch.float32
    np.testing.assert_array_equal(t.cpu().numpy(), z)


def test_empty_and_degenerate_rasters(xb):
    for shape in ((0, 0), (1, 1), (1, 7), (5, 1), (2, 2)):
        z = np.arange(shape[0] * shape[1], dtype=np.float32).reshape(shape)
        out = host(xb.slope(da(xb, dev(z))))
        assert out.shape == shape and np.isnan(out).all()
        m = host(xb.mean(da(xb, dev(z))))
        assert m.shape == shape
        if z.size:
            assert_close_f32(m, o.focal_mean(z), atol=0)


def test_large_zonal_blocks_and_scatter(xb):
    """1024 zones as a 32x32 block grid and as a scattered hash (SURVEY.md 8d zones)."""
    rng = np.random.default_rng(7)
    H = W = 1024
    values = terrain(rng, H, W, nans=0.001)
    yy, xx = np.mgrid[0:H, 0:W]
    for zones in (((yy // 32) * 32 + xx // 32).astype(np.int32),
                  ((yy * 7919 + xx * 104729) % 1024).astype(np.int32)):
        df = xb.zonal_stats(da(xb, dev(zones)), da(xb, dev(values)))
        ref = o.zonal_stats(zones, values)
        np.testing.assert_array_equal(np.asarray(df["zone"]), ref["zone"])
        np.testing.assert_array_equal(np.asarray(df["count"]), ref["count"])
        np.testing.assert_array_equal(np.asarray(df["min"]), ref["min"])
        np.testing.assert_array_equal(np.asarray(df["max"]), ref["max"])
        for c in ("mean", "sum", "std", "var"):
            np.testing.assert_allclose(np.asarray(df[c]), ref[c], rtol=1e-5, err_msg=c)


def test_row_stripes_are_partition_invariant(xb):
    """SURVEY.md 8e: an N-stripe result must equal the single-raster result bit for bit.  The
    stripes (with 1-row halos cut from the full raster, as the NCCL exchange would deliver
    them) are processed one after the other on this GPU."""
    from xrspatial_b200.stripes import split_rows
    rng = np.random.default_rng(21)
    z = terrain(rng, 1000, 768, nans=0.002)
    full = dev(z)
    ops = {"slope": xb.slope, "aspect": xb.aspect, "curvature": xb.curvature, "hillshade": xb.hillshade,
           "mean": xb.mean}
    whole = {k: host(f(da(xb, full))) for k, f in ops.items()}
    for world in (2, 3, 8):
        parts = {k: [] for k in ops}
        for (y0, y1) in split_rows(z.shape[0], world):
            top = 1 if y0 > 0 else 0
            bot = 1 if y1 < z.shape[0] else 0
            stripe = full[y0 - top:y1 + bot].contiguous()
            for k, f in ops.items():
                out = f(da(xb, stripe)).data
                parts[k].append(out[top:top + (y1 - y0)].cpu().numpy())
        for k in ops:
            np.testing.assert_array_equal(np.concatenate(parts[k]), whole[k], err_msg="%s world=%d" % (k, world))


def _stripe_worker(rank, world, port, H, W, q):
    import os
    import sys
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import torch.distributed as dist
    import xrspatial_b200 as xbm
    from xrspatial_b200.stripes import RowStripes
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        rng = np.random.default_rng(33)
        z = terrain(rng, H, W, nans=0.002)
        zones = ((np.arange(H)[:, None] // 64) * 8 + np.arange(W)[None, :] // 64).astype(np.int32)
        dev_ = torch.device("cuda", rank)
        st = RowStripes(H, W, radius=1, device=dev_)
        st.interior.copy_(torch.from_numpy(z[st.y0:st.y1]))
        res = {}
        attrs = {"res": (30.0, 30.0)}
        for name, fn in (("slope", xbm.slope), ("hillshade", xbm.hillshade), ("mean", xbm.mean)):
            res[name] = st.apply(fn, attrs=attrs).cpu().numpy()                       # overlapped exchange
            res[name + "/plain"] = st.apply(fn, attrs=attrs, overlap=False).cpu().numpy()
        res["mean3"] = st.mean(passes=3).cpu().numpy()                                 # one exchange per pass
        krng = np.random.default_rng(8)
        for k in (9, 25):                                                              # wide halos (r = 4, 12)
            kern = krng.standard_normal((k, k))
            sk = RowStripes(H, W, radius=k // 2, device=dev_)
            sk.interior.copy_(torch.from_numpy(z[sk.y0:sk.y1]))
            res["conv%d" % k] = sk.convolve(kern).cpu().numpy()
            res["conv%d/plain" % k] = sk.convolve(kern, overlap=False).cpu().numpy()
        st.exchange()
        zagg = xbm.DataArray(torch.from_numpy(zones[st.y0:st.y1]).cuda(), dims=("y", "x"))
        vagg = xbm.DataArray(st.interior, dims=("y", "x"))
        df = xbm.zonal_stats(zagg, vagg, comm=dist.group.WORLD)
        q.put((rank, st.y0, st.y1, res, {c: np.asarray(df[c]) for c in df.columns}))
    finally:
        dist.destroy_process_group()


def test_two_gpu_stripes_match_single_gpu(xb):
    """Real NCCL halo exchange + zonal all-gather merge on 2 GPUs (skipped on 1-GPU boxes)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import socket
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    H, W = 600, 512
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_stripe_worker, args=(r, 2, port, H, W, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = sorted([q.get(timeout=300) for _ in range(2)], key=lambda t: t[0])
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    rng = np.random.default_rng(33)
    z = terrain(rng, H, W, nans=0.002)
    zones = ((np.arange(H)[:, None] // 64) * 8 + np.arange(W)[None, :] // 64).astype(np.int32)
    agg = da(xb, dev(z))
    for name, fn in (("slope", xb.slope), ("hillshade", xb.hillshade), ("mean", xb.mean)):
        whole = host(fn(agg))
        for variant in (name, name + "/plain"):
            stitched = np.concatenate([g[3][variant] for g in got])
            np.testing.assert_array_equal(stitched, whole, err_msg=variant)
    # focal.mean(passes=3): one halo exchange per pass (focal.py:72-75, 258-259)
    np.testing.assert_array_equal(np.concatenate([g[3]["mean3"] for g in got]), host(xb.mean(agg, passes=3)),
                                  err_msg="mean passes=3")
    # k = 9 / 25 convolutions over stripes with 4- / 12-row halos
    krng = np.random.default_rng(8)
    for k in (9, 25):
        kern = krng.standard_normal((k, k))
        whole = host(xb.convolution_2d(agg, kern))
        for variant in ("conv%d" % k, "conv%d/plain" % k):
            np.testing.assert_array_equal(np.concatenate([g[3][variant] for g in got]), whole, err_msg=variant)
    df = xb.zonal_stats(da(xb, dev(zones)), agg)
    for c in df.columns:
        a, b = np.asarray(df[c]), got[0][4][c]
        if c in ("zone", "count", "min", "max"):
            np.testing.assert_array_equal(a, b, err_msg=c)
        else:
            np.testing.assert_allclose(a, b, rtol=1e-9, equal_nan=True, err_msg=c)


def test_zonal_majority(xb, known, refout):
    # ties -> smallest value (test_zonal.py:567-590)
    zones = np.array([[1, 1, 1, 1], [1, 1, 2, 2], [2, 2, 2, 2]], dtype=np.int32)
    values = np.array([[1, 1, 2, 2], [3, 3, 5, 5], [5, 5, 6, 6]], dtype=np.float32)
    df = xb.zonal_stats(da(xb, dev(zones)), da(xb, dev(values)), stats_funcs=["majority"])
    np.testing.assert_array_equal(np.asarray(df["zone"]), [1, 2])
    np.testing.assert_array_equal(np.asarray(df["majority"]), [1, 5])
    # test_zonal.py:61-75 default table incl. majority (float zones with a NaN, inf / NaN values)
    df = xb.zonal_stats(da(xb, dev(known["zonal.data_zones"])), da(xb, dev(known["zonal.data_values_2d"])),
                        stats_funcs=["mean", "max", "min", "sum", "std", "var", "count", "majority"])
    for c in ("zone", "mean", "max", "min", "sum", "std", "var", "count", "majority"):
        np.testing.assert_allclose(np.asarray(df[c], dtype=np.float64), known["zonal.result_default_stats." + c],
                                   rtol=1e-5, atol=1e-7, err_msg=c)
    # continuous values: every value unique -> majority is the zone minimum (reference output)
    df = xb.zonal_stats(da(xb, dev(refout["zonal.zones_i32"])), da(xb, dev(refout["zonal.values_f32"])),
                        stats_funcs=["majority", "count"])
    np.testing.assert_array_equal(np.asarray(df["majority"]), refout["zonal.f32_i32.majority"])
    # categorical raster vs the oracle
    rng = np.random.default_rng(9)
    zc = rng.integers(0, 37, size=(300, 256)).astype(np.int32)
    vc = rng.integers(0, 9, size=(300, 256)).astype(np.float32)
    vc[rng.random(vc.shape) < 0.01] = np.nan
    df = xb.zonal_stats(da(xb, dev(zc)), da(xb, dev(vc)), stats_funcs=["majority"])
    ref = o.zonal_stats(zc, vc, stats_funcs=["majority"])
    np.testing.assert_array_equal(np.asarray(df["majority"]), ref["majority"])


# ----------------------------------------------------------------- BASELINE.json full sizes
def _interior(t):
    return t[1:-1, 1:-1]


@pytest.mark.parametrize("side", [32768, 65536])
def test_full_size_properties(xb, side):
    """Size-independent properties at the benchmark sizes (32768^2 = configs[1], 65536^2 = the
    striped raster of configs[4]); the oracle cannot run here in seconds, closed forms can."""
    import math
    torch.cuda.empty_cache()         # what earlier tests left in torch's cache is free for this one
    free, _ = torch.cuda.mem_get_info()
    if free < side * side * 4 * 4:      # at most three rasters are alive at once
        pytest.skip("not enough device memory for a %d^2 raster" % side)
    H = W = side
    ys = torch.arange(H, device="cuda", dtype=torch.float32)[:, None]
    xs = torch.arange(W, device="cuda", dtype=torch.float32)[None, :]
    ramp = (0.5 * xs + 0.25 * ys).contiguous()          # exact in float32
    agg = da(xb, ramp, res=(30.0, 30.0))
    # planar ramp: Horn slope is the same constant in every interior cell, aspect likewise
    s = xb.slope(agg).data
    expect = math.degrees(math.atan(math.hypot(0.5 / 30.0, 0.25 / 30.0))) * (57.29578 / (180 / math.pi))
    si = _interior(s)
    assert float(si.min()) == float(si.max())
    assert abs(float(si[0, 0]) - expect) <= 1e-5 * expect
    assert bool(torch.isnan(s[0]).all() and torch.isnan(s[-1]).all() and torch.isnan(s[:, 0]).all()
                and torch.isnan(s[:, -1]).all())
    del s, si
    a = xb.aspect(agg).data
    ai = _interior(a)
    exp_a = (math.degrees(math.atan2(-0.5 * 8, 0.25 * 8)) + 360.0) % 360.0   # atan2(-X, Y), X = 8*0.5, Y = 8*0.25
    assert float(ai.min()) == float(ai.max()) and abs(float(ai[0, 0]) - exp_a) <= 1e-4
    del a, ai
    # a plane has zero curvature (-0.0 like the reference's flat case)
    c = _interior(xb.curvature(agg).data)
    lo, hi = torch.aminmax(c)
    assert float(lo) == 0.0 and float(hi) == 0.0
    del c
    # focal.mean: interior mean of a plane is the plane itself; window counts on the border are
    # 6 (edges) and 4 (corners): check through the constant raster too
    m = xb.mean(agg).data
    lo, hi = torch.aminmax(_interior(m.sub_(ramp)))
    assert max(-float(lo), float(hi)) <= 1e-3 * 1e-2   # exact up to f32 rounding of the mean
    del m
    ramp.fill_(7.25)
    const = da(xb, ramp, res=(30.0, 30.0))
    m = xb.mean(const).data
    assert float(m.min()) == 7.25 and float(m.max()) == 7.25          # idempotent on constants, clamped edges
    del m
    h = _interior(xb.hillshade(const).data)
    flat = 0.5 * (math.sin(math.radians(25)) + 1.0)
    assert float(h.min()) == float(h.max()) and abs(float(h[0, 0]) - flat) < 1e-6
    del h
    # partition invariance at full size: rows [a, b) of the whole-raster result == the result of
    # the stripe [a-1, b+1) computed on its own
    for r0 in range(0, H, 4096):     # in row blocks: the expression's temporaries are raster-sized
        y = ys[r0:r0 + 4096]
        ramp[r0:r0 + 4096].copy_(torch.sin(xs * 0.001) * 400 + torch.cos(y * 0.0007) * 300 + 0.01 * ((xs * 7 + y * 13) % 97))
    whole = xb.slope(agg).data
    a0, b0 = H // 2 - 1000, H // 2 + 1000
    part = xb.slope(da(xb, ramp[a0 - 1:b0 + 1], res=(30.0, 30.0))).data[1:-1]
    assert bool(torch.equal(torch.nan_to_num(whole[a0:b0], nan=-5.0), torch.nan_to_num(part, nan=-5.0)))


def test_full_size_box_and_zonal_properties(xb):
    """The running box (convolve_2d with uniform taps, focal.apply mean over all-ones windows) and the zonal
    group-by at the benchmark size 32768^2, through properties that need no oracle: the mean of a plane over a
    symmetric window is the plane's value at the window's centre; a constant stays a constant under clamped
    NaN-skipping windows; block zones of a plane have closed-form counts, means, minima and maxima."""
    from xrspatial_b200 import focal
    from xrspatial_b200.convolution import convolve_2d
    side = 32768
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < side * side * 4 * 5:
        pytest.skip("not enough device memory for a %d^2 raster" % side)
    ys = torch.arange(side, device="cuda", dtype=torch.float32)[:, None]
    xs = torch.arange(side, device="cuda", dtype=torch.float32)[None, :]
    ramp = (0.5 * xs + 0.25 * ys).contiguous()          # exact in float32, < 2^15
    for k in (9, 25):
        r = k // 2
        out = convolve_2d(ramp, np.ones((k, k)) / (k * k))
        assert used_tma(xb) == 3
        inner = out[r:-r, r:-r]
        assert float((inner - ramp[r:-r, r:-r]).abs().max()) <= 1e-5 * 24576.0     # the window's centre value
        assert bool(torch.isnan(out[:r]).all() and torch.isnan(out[-r:]).all() and torch.isnan(out[:, :r]).all()
                    and torch.isnan(out[:, -r:]).all())                              # the reference's NaN ring
        assert not bool(torch.isnan(inner).any())
        del out, inner
    m = focal.apply(da(xb, ramp), np.ones((5, 5))).data
    assert used_tma(xb) == 3
    assert float((m[2:-2, 2:-2] - ramp[2:-2, 2:-2]).abs().max()) <= 1e-5 * 24576.0
    # clamped corner window: rows 0..2 x columns 0..2 of the plane -> its value at (1, 1)
    assert abs(float(m[0, 0]) - 0.75) <= 1e-6 and not bool(torch.isnan(m).any())
    del m
    # block zones of the plane: 32 x 32 blocks of 1024 x 1024 cells
    zones = ((ys.to(torch.int32) // 1024) * 32 + (xs.to(torch.int32) // 1024)).contiguous()
    df = xb.zonal_stats(da(xb, zones), da(xb, ramp), stats_funcs=["mean", "max", "min", "count", "sum"])
    zid = np.asarray(df["zone"])
    assert np.array_equal(zid, np.arange(1024))
    by, bx = zid // 32, zid % 32
    assert np.array_equal(np.asarray(df["count"]), np.full(1024, 1024.0 * 1024.0))
    lo = 0.5 * (bx * 1024) + 0.25 * (by * 1024)
    hi = 0.5 * (bx * 1024 + 1023) + 0.25 * (by * 1024 + 1023)
    assert np.array_equal(np.asarray(df["min"]), lo) and np.array_equal(np.asarray(df["max"]), hi)
    np.testing.assert_allclose(np.asarray(df["mean"]), 0.5 * (lo + hi), rtol=1e-12)       # exact sums of a plane
    np.testing.assert_allclose(np.asarray(df["sum"]), 0.5 * (lo + hi) * 1024.0 * 1024.0, rtol=1e-12)
    # a categorical raster with a known majority: class = block row parity, except a minority stripe
    ramp.copy_(((ys.to(torch.int32) // 1024) % 2).to(torch.float32).expand(side, side))
    ramp[:, ::7] = 5.0
    df = xb.zonal_stats(da(xb, zones), da(xb, ramp), stats_funcs=["majority"])
    assert np.array_equal(np.asarray(df["majority"]), (by % 2).astype(np.float64))


def test_hotspots_vs_reference_outputs(xb, refout):
    r = refout
    agg = da(xb, dev(r["hotspots.dem"]))
    out = xb.hotspots(agg, r["hotspots.kernel"])
    assert out.attrs["unit"] == "%" and out.data.dtype == torch.int8
    np.testing.assert_array_equal(host(out), r["hotspots.out"])
    np.testing.assert_array_equal(host(xb.hotspots(agg, np.ones((5, 5)))), r["hotspots.out_5x5"])
    outh = xb.hotspots(da(xb, r["hotspots.dem"]), r["hotspots.kernel"]).data     # numpy in -> numpy out
    assert isinstance(outh, np.ndarray) and outh.dtype == np.int8
    np.testing.assert_array_equal(outh, r["hotspots.out"])
    with pytest.raises(ZeroDivisionError):                                        # test_focal.py:457-463
        xb.hotspots(da(xb, dev(np.zeros((10, 12), np.float32))), np.ones((3, 3)))


def test_crosstab_vs_reference_outputs(xb, refout):
    r = refout
    zones, values = da(xb, dev(r["crosstab.zones"])), da(xb, dev(r["crosstab.values"]))
    for agg_name in ("count", "percentage"):
        df = xb.zonal_crosstab(zones, values, agg=agg_name)
        np.testing.assert_array_equal(np.asarray([float(c) for c in df.columns[1:]]), r["crosstab.%s.columns" % agg_name])
        np.testing.assert_allclose(np.asarray(df.values, dtype=np.float64), r["crosstab.%s.table" % agg_name],
                                   rtol=1e-6, equal_nan=True)
    df = xb.zonal_crosstab(zones, values, zone_ids=[1, 3, 9], cat_ids=[11.0, 13.0], nodata_values=12.0)
    np.testing.assert_array_equal(np.asarray(df.values, dtype=np.float64), r["crosstab.sub.table"])
    with pytest.raises(ValueError):
        xb.zonal_crosstab(zones, values, agg="median")


def test_geodesic_vs_reference_outputs(xb, refout):
    r = refout
    z = r["geodesic.dem"]

    def grid(data, lat, lon, two_d=False):
        g = xb.DataArray(data, dims=("lat", "lon"))
        if two_d:
            g.coords["latitude"], g.coords["longitude"] = lat, lon
        else:
            g["lat"], g["lon"] = lat, lon
        return g

    tol = dict(rtol=1e-5, atol=1e-6)
    for data in (dev(z), dev(z.astype(np.float32))):       # float64 and float32 elevation
        g = grid(data, r["geodesic.lat"], r["geodesic.lon"])
        s = host(xb.slope(g, method="geodesic"))
        assert s.dtype == np.float32
        if data.dtype == torch.float32:
            # the golden is of the float64 DEM: float32 cells are held to the bound of their own values
            ex = expect(z.astype(np.float32), r["geodesic.lat"], r["geodesic.lon"])
            check(s, ex, "golden grid float32")
            check(host(xb.aspect(g, method="geodesic")), ex, "golden grid float32", aspect=True)
        else:
            np.testing.assert_allclose(s, r["geodesic.slope"], equal_nan=True, **tol)
            np.testing.assert_allclose(host(xb.slope(g, method="geodesic", z_unit="foot")), r["geodesic.slope_ft"],
                                       equal_nan=True, **tol)
            a = host(xb.aspect(g, method="geodesic"))
            ref = r["geodesic.aspect"]
            np.testing.assert_array_equal(np.isnan(a), np.isnan(ref))
            np.testing.assert_array_equal(a == -1, ref == -1)
            m = ~np.isnan(ref) & (ref != -1)
            d = np.abs(a[m] - ref[m])
            assert np.minimum(d, 360 - d).max() < 1e-3
            g2 = grid(data, r["geodesic.lat2d"], r["geodesic.lon2d"], two_d=True)
            np.testing.assert_allclose(host(xb.slope(g2, method="geodesic")), r["geodesic.slope_2d"], equal_nan=True,
                                       **tol)
            a2 = host(xb.aspect(g2, method="geodesic"))
            ref2 = r["geodesic.aspect_2d"]
            m = ~np.isnan(ref2) & (ref2 != -1)
            d = np.abs(a2[m] - ref2[m])
            assert np.minimum(d, 360 - d).max() < 1e-3
    # numpy in -> numpy out
    gh = grid(z, r["geodesic.lat"], r["geodesic.lon"])
    sh = xb.slope(gh, method="geodesic").data
    assert isinstance(sh, np.ndarray)
    np.testing.assert_allclose(sh, r["geodesic.slope"], rtol=1e-5, atol=1e-6, equal_nan=True)
    # larger regular grid vs the oracle
    rng = np.random.default_rng(4)
    zz = terrain(rng, 300, 400).astype(np.float64)
    lat, lon = np.linspace(40.0, 39.5, 300), np.linspace(-105.0, -104.2, 400)
    ref = o.geodesic(zz, np.broadcast_to(lat[:, None], zz.shape), np.broadcast_to(lon[None, :], zz.shape), nthreads=8)
    got = host(xb.slope(grid(dev(zz), lat, lon), method="geodesic"))
    np.testing.assert_allclose(got, ref, rtol=1e-5, atol=1e-6, equal_nan=True)


def test_pitched_and_ragged_inputs(xb):
    """Row pitch > W (a column slice of a wider raster), widths that are not a multiple of 4 or of
    the 128-cell strip, and a misaligned base pointer all give the oracle's values."""
    rng = np.random.default_rng(17)
    big = terrain(rng, 260, 1100, nans=0.003)
    t = dev(big)
    for (x0, x1) in ((0, 1024), (4, 1028), (8, 524), (0, 1099), (3, 770), (128, 131)):
        view = t[:, x0:x1]                       # pitch 1100 * 4 bytes, not contiguous
        ref_in = big[:, x0:x1]
        got = host(xb.slope(da(xb, view)))
        assert_close_f32(got, o.slope(ref_in, 30.0, 30.0, nthreads=8), what="slope view %d:%d" % (x0, x1))
        assert_close_f32(host(xb.mean(da(xb, view))), o.focal_mean(ref_in, nthreads=8), atol=0,
                         what="mean view %d:%d" % (x0, x1))
    # W = 1100 (multiple of 4, not of 128): TMA path with a ragged last strip
    assert_close_f32(host(xb.hillshade(da(xb, t))), o.hillshade(big, nthreads=8), what="hillshade 1100")
    assert used_tma(xb) == 1
    # negative cell size in y (descending coordinates, utils.py:204-230): slope squares it
    agg = xb.DataArray(t, dims=("y", "x"))
    agg["y"] = np.linspace(260 * 30.0, 30.0, 260)
    agg["x"] = np.linspace(0.0, 1099 * 30.0, 1100)
    assert_close_f32(host(xb.slope(agg)), o.slope(big, 30.0, -30.0, nthreads=8), what="negative cellsize_y")


def test_ragged_widths_every_strip_operator(xb):
    """Widths TMA cannot describe (W % 4 != 0) go through the cp.async ring with transposed,
    coalesced 4-byte stores: every operator of the skeleton, single- and multi-output, f32 and f64."""
    rng = np.random.default_rng(23)
    for (h, w) in ((70, 131), (129, 257), (40, 1023), (33, 5)):
        z = terrain(rng, h, w, nans=0.01)
        agg = da(xb, dev(z))
        assert_close_f32(host(xb.slope(agg)), o.slope(z, 30.0, 30.0, nthreads=4), what="slope %dx%d" % (h, w))
        assert used_tma(xb) == 0
        assert_aspect_close(host(xb.aspect(agg)), o.aspect(z, nthreads=4), what="aspect %dx%d" % (h, w))
        ref_c = o.curvature(z, 30.0, nthreads=4)
        assert_close_f32(host(xb.curvature(agg)), ref_c, atol=1e-6 * max(np.nanmax(np.abs(ref_c)), 1e-30),
                         what="curvature %dx%d" % (h, w))
        assert_close_f32(host(xb.hillshade(agg)), o.hillshade(z, nthreads=4), what="hillshade %dx%d" % (h, w))
        assert_close_f32(host(xb.mean(agg)), o.focal_mean(z, nthreads=4), atol=0, what="mean %dx%d" % (h, w))
        m64 = host(xb.mean(da(xb, dev(z.astype(np.float64)))))
        assert m64.dtype == np.float64
        np.testing.assert_allclose(m64, o.focal_mean(z.astype(np.float64), nthreads=4), rtol=1e-12, equal_nan=True)
        suite = xb.surface_suite(agg)
        for name in ("slope", "curvature", "hillshade"):
            np.testing.assert_array_equal(host(suite[name]), host(getattr(xb, name)(agg)), err_msg="suite " + name)
        np.testing.assert_array_equal(host(suite["aspect"]), host(xb.aspect(agg)))


def test_integer_and_f64_inputs_are_cast_like_the_reference(xb):
    # tests/test_slope.py:70-79 parametrises over int32/int64/uint32/uint64/float32/float64
    base = np.random.default_rng(2841).integers(-100, 100, size=(10, 15))
    ref = o.slope(base.astype(np.float32), 1, 1)
    for dt in (np.int32, np.int64, np.float32, np.float64):
        got = host(xb.slope(da(xb, dev(base.astype(dt)), res=(1, 1))))
        assert got.dtype == np.float32
        assert_close_f32(got, ref, what=str(dt))
        goth = xb.slope(da(xb, base.astype(dt), res=(1, 1))).data
        assert_close_f32(goth, ref, what="host " + str(dt))
    for dt in (np.uint8, np.uint16):
        got = host(xb.ndvi(da(xb, dev(np.array([[1, 1], [1, 1]], dtype=dt))),
                           da(xb, dev(np.array([[0, 2], [1, 2]], dtype=dt)))))
        np.testing.assert_allclose(got, [[1, -0.33333334], [0, -0.33333334]], rtol=1e-6)


@pytest.mark.parametrize("dt", [np.int16, np.uint16, np.int32, np.float64])
def test_direct_ingest_matches_cast_then_compute(xb, dt):
    """int16 / uint16 / int32 / float64 rasters are read directly (xrs_surface_typed) and must give
    exactly what the float32 kernels give on the `.astype(float32)` copy (slope.py:58,150)."""
    rng = np.random.default_rng(31)
    base = terrain(rng, 300, 512) - (1500.0 if np.issubdtype(dt, np.signedinteger) or dt == np.float64 else 0.0)
    if dt == np.float64:
        raw = base.astype(np.float64) * 1.000000123          # not exactly representable in f32
    else:
        raw = np.round(base).astype(dt)
    f32 = raw.astype(np.float32)
    for name, fn, kw in (("slope", xb.slope, {}), ("aspect", xb.aspect, {}), ("curvature", xb.curvature, {}),
                         ("hillshade", xb.hillshade, dict(azimuth=300, angle_altitude=40))):
        ref = host(fn(da(xb, dev(f32)), **kw))
        got = fn(da(xb, dev(raw)), **kw)
        assert used_tma(xb) == 2, "direct-ingest kernel was not selected for %s" % np.dtype(dt).name
        assert got.data.dtype == torch.float32
        np.testing.assert_array_equal(host(got), ref, err_msg="%s %s" % (name, np.dtype(dt).name))
        goth = fn(da(xb, raw), **kw).data                    # host raster: raw cells cross PCIe
        assert isinstance(goth, np.ndarray) and goth.dtype == np.float32
        np.testing.assert_array_equal(goth, ref, err_msg="host %s %s" % (name, np.dtype(dt).name))
    # layouts the ingest path does not take fall back to cast + float32 kernels, same values
    odd = raw[:, :509]
    np.testing.assert_array_equal(host(xb.slope(da(xb, dev(odd)))), host(xb.slope(da(xb, dev(odd.astype(np.float32))))))
    np.testing.assert_array_equal(xb.slope(da(xb, np.ascontiguousarray(odd))).data,
                                  host(xb.slope(da(xb, dev(odd.astype(np.float32))))))


# ----------------------------------------------------------------- round 2: drop-in contract
def test_zonal_default_stats_are_the_references(xb, known):
    """zonal.py:422-436: the default `stats_funcs` list includes `majority`."""
    zones, values = known["zonal.data_zones"], known["zonal.data_values_2d"]
    for mk in (dev, lambda a: a):   # device raster, numpy raster
        df = xb.zonal_stats(da(xb, mk(zones)), da(xb, mk(values)))
        assert list(df.columns) == ["zone", "mean", "max", "min", "sum", "std", "var", "count", "majority"]
        for c in df.columns:
            np.testing.assert_allclose(np.asarray(df[c], dtype=np.float64), known["zonal.result_default_stats." + c],
                                       rtol=1e-5, atol=1e-7, err_msg=c)


def test_zonal_custom_stats(xb, known, refout):
    """test_zonal.py:204-246 / :497-545: `stats_funcs` as a dict of callables, nodata 0, zone_ids [1, 2];
    then the reference's own per-zone loop on a seeded raster (reference_outputs.npz)."""
    custom = {"double_sum": lambda v: v.sum() * 2, "range": lambda v: v.max() - v.min()}
    zones, values = known["zonal.data_zones"], known["zonal.data_values_2d"]
    zid = known["zonal.result_custom_stats.zone_ids"].tolist()
    nod = known["zonal.result_custom_stats.nodata_values"].item()
    for mk in (dev, lambda a: a):
        df = xb.zonal_stats(da(xb, mk(zones)), da(xb, mk(values)), zone_ids=zid, stats_funcs=custom,
                            nodata_values=nod)
        assert list(df.columns) == ["zone", "double_sum", "range"]
        for c in df.columns:
            np.testing.assert_allclose(np.asarray(df[c], dtype=np.float64), known["zonal.result_custom_stats." + c],
                                       rtol=1e-5, atol=1e-7, err_msg=c)
        arr = xb.zonal_stats(da(xb, mk(zones)), da(xb, mk(values)), zone_ids=zid, stats_funcs=custom,
                             nodata_values=nod, return_type="xarray.DataArray")
        assert arr.dims == ("stats", "y", "x") and list(arr.coords["stats"]) == ["double_sum", "range"]
        np.testing.assert_allclose(host(arr), known["zonal.result_custom_stats_dataarray"], equal_nan=True)
    # a dict keyed by a built-in name runs the CALLABLE, never the built-in (reference: zonal.py:640-642)
    df = xb.zonal_stats(da(xb, dev(zones)), da(xb, dev(values)), zone_ids=zid, nodata_values=nod,
                        stats_funcs={"mean": lambda v: 42.0})
    np.testing.assert_array_equal(np.asarray(df["mean"]), [42.0, 42.0])
    with pytest.raises(ValueError):
        xb.zonal_stats(da(xb, dev(zones)), da(xb, dev(values)), stats_funcs={"mean": "mean"})
    # seeded raster, three callables, zone filter incl. a missing id, nodata
    r = refout
    custom3 = {"double_sum": lambda v: v.sum() * 2, "range": lambda v: v.max() - v.min(),
               "l2norm": lambda v: float(np.sqrt(np.sum(np.asarray(v.cpu() if hasattr(v, "cpu") else v, dtype=np.float64) ** 2)))}
    for mk in (dev, lambda a: a):
        df = xb.zonal_stats(da(xb, mk(r["zonal.zones_i32"])), da(xb, mk(r["zonal.values_f32"])),
                            zone_ids=[3, 7, 100, 999], stats_funcs=custom3, nodata_values=0.0)
        np.testing.assert_array_equal(np.asarray(df["zone"]), r["zonal.f32_i32_custom.zone"])
        for c in ("double_sum", "range", "l2norm"):
            np.testing.assert_allclose(np.asarray(df[c], dtype=np.float64), r["zonal.f32_i32_custom." + c],
                                       rtol=2e-6, err_msg=c)


def test_majority_by_sort_equals_the_pair_table(xb, monkeypatch):
    """`majority` has two engines: the (zone, value) pair-count kernel (int32 zones, float32-exact
    values) and one device sort (everything else: wide / non-integer zone ids, float64 values,
    continuous rasters that overflow the pair table).  Same answers, incl. NaN, nodata and -0.0."""
    from xrspatial_b200 import zonal as Z
    rng = np.random.default_rng(4)
    zc = rng.integers(-3, 40, size=(257, 300)).astype(np.int32)
    vc = rng.integers(-4, 9, size=(257, 300)).astype(np.float32)
    vc[rng.random(vc.shape) < 0.02] = np.nan
    zero = vc == 0
    vc[zero] = np.where(rng.random(zero.sum()) < 0.5, -0.0, 0.0).astype(np.float32)
    uz = np.unique(zc)
    for nod in (None, 3.0):
        ref = o.zonal_stats(zc, vc, stats_funcs=["majority"], nodata_values=nod)
        np.testing.assert_array_equal(ref["zone"], uz)
        a = Z.majority_by_zone(dev(zc), dev(vc), uz, nod)                       # pair table
        b = Z.majority_by_zone(dev(zc.astype(np.int64)), dev(vc), uz, nod)      # sort, float32 keys
        c = Z.majority_by_zone(dev(zc.astype(np.float64)), dev(vc.astype(np.float64)), uz.astype(np.float64), nod)
        for got in (a, b, c):
            np.testing.assert_array_equal(got, np.asarray(ref["majority"], dtype=np.float64))
    # float64 values that float32 cannot hold + non-integer zone ids (rank keys)
    v64 = (rng.integers(0, 7, size=(64, 128)) * 0.1 + 1e6).astype(np.float64)
    z64 = (rng.integers(0, 5, size=(64, 128)) * 0.5 - 1.0).astype(np.float64)
    z64[0, :5] = np.nan
    ref = o.zonal_stats(z64, v64, stats_funcs=["majority"])
    got = Z.majority_by_zone(dev(z64), dev(v64), np.asarray(ref["zone"]))
    np.testing.assert_array_equal(got, np.asarray(ref["majority"], dtype=np.float64))
    # continuous values through the public API: the pair table overflows its (small here) budget
    vals = rng.standard_normal((64, 4096)).astype(np.float32)
    zz = (np.arange(64)[:, None] // 16 * 2 + np.arange(4096)[None, :] // 2048).astype(np.int32)
    monkeypatch.setattr(Z, "_PAIR_CAP", 1 << 10)
    monkeypatch.setattr(Z, "_MAJORITY_PAIR_MAX_CAP", 1 << 12)
    sorts = []
    by_sort = Z._majority_by_sort
    monkeypatch.setattr(Z, "_majority_by_sort", lambda *a: sorts.append(a[2]) or by_sort(*a))
    df = xb.zonal_stats(da(xb, dev(zz)), da(xb, dev(vals)), stats_funcs=["majority"])
    assert sorts == [8], "the pair table did not overflow into the sort"
    ref = o.zonal_stats(zz, vals, stats_funcs=["majority"])
    np.testing.assert_array_equal(np.asarray(df["majority"]), np.asarray(ref["majority"], dtype=np.float64))


def test_summarize_terrain_docstring_example(xb):
    """analytics.py:29-71: the docstring's 5 x 8 raster and its slope / curvature / aspect tables, for a
    device raster and a numpy raster; variables are added with `ds[name] = ...` (a read-only `data_vars`)."""
    data = np.zeros((5, 8), dtype=np.float64)
    data[2, 2], data[2, 5] = 1, -1
    nan = np.nan
    slope = np.array([[nan] * 8,
                      [nan, 10.024988, 14.036243, 10.024988, 10.024988, 14.036243, 10.024988, nan],
                      [nan, 14.036243, 0., 14.036243, 14.036243, 0., 14.036243, nan],
                      [nan, 10.024988, 14.036243, 10.024988, 10.024988, 14.036243, 10.024988, nan],
                      [nan] * 8])
    curv = np.array([[nan] * 8,
                     [nan, -0., -100., -0., -0., 100., -0., nan],
                     [nan, -100., 400., -100., 100., -400., 100., nan],
                     [nan, -0., -100., -0., -0., 100., -0., nan],
                     [nan] * 8])
    aspect = np.array([[nan] * 8,
                       [nan, 315., 0., 45., 135., 180., 225., nan],
                       [nan, 270., -1., 90., 90., -1., 270., nan],
                       [nan, 225., 180., 135., 45., 0., 315., nan],
                       [nan] * 8])
    for mk in (dev, lambda a: a):
        raster = xb.DataArray(mk(data), name="myraster", attrs={"res": (1, 1)})
        ds = xb.summarize_terrain(raster)
        assert list(ds.data_vars) == ["myraster", "myraster-slope", "myraster-curvature", "myraster-aspect"]
        with pytest.raises(TypeError):
            ds.data_vars["x"] = raster           # read-only, like xarray
        assert_close_f32(host(ds["myraster-slope"]), slope, what="slope")
        assert_close_f32(host(ds["myraster-curvature"]), curv, atol=1e-4, what="curvature")
        assert_aspect_close(host(ds["myraster-aspect"]), aspect, what="aspect")
        assert ds["myraster-slope"].attrs == {"res": (1, 1)} and ds["myraster-slope"].dims == raster.dims
    with pytest.raises(NameError):
        xb.summarize_terrain(xb.DataArray(dev(data)))


def test_aspect_of_a_nodata_pixel_on_a_plateau(xb):
    """aspect.py:74-88: the W / E / N / S neighbours of an isolated NaN on a flat area are NaN, not -1
    (one Horn sum is NaN, the other 0); single kernel, fused suite and typed ingestion alike."""
    z = np.full((40, 256), 250.0, dtype=np.float32)
    z[17, 101] = np.nan
    z[30, 5] = np.nan
    z[3:6, 200:203] = 260.0
    ref = o.aspect(z)
    assert np.isnan(ref[17, 100]) and np.isnan(ref[16, 101]) and ref[10, 10] == -1
    assert_aspect_close(host(xb.aspect(da(xb, dev(z)))), ref, what="aspect")
    assert_aspect_close(host(xb.surface_suite(da(xb, dev(z)))["aspect"]), ref, what="suite aspect")
    z64 = z.astype(np.float64)
    assert_aspect_close(host(xb.aspect(da(xb, dev(z64)))), o.aspect(z64.astype(np.float32)), what="f64 ingest")
    assert_aspect_close(xb.aspect(da(xb, z)).data, ref, what="host path")


def test_bare_dataarray_without_coords_uses_unit_cells(xb):
    """utils.py:233-277: no attrs['res'] and no coordinates -> xarray's default integer index -> cellsize 1."""
    rng = np.random.default_rng(12)
    z = terrain(rng, 64, 128)
    agg = xb.DataArray(dev(z), dims=("y", "x"))
    assert_close_f32(host(xb.slope(agg)), o.slope(z, 1.0, 1.0), what="slope")
    assert_close_f32(host(xb.curvature(agg)), o.curvature(z, 1.0), atol=1e-6 * np.nanmax(np.abs(o.curvature(z, 1.0))),
                     what="curvature")


def test_pinned_cache_is_bounded_and_lru(xb):
    """_hostmem: idle page-locked blocks are capped; the least recently released go first."""
    from xrspatial_b200 import _hostmem as hm
    hm.trim()
    old = hm.MAX_CACHED_BYTES
    hm.MAX_CACHED_BYTES = 3 << 20
    try:
        for mb in (1, 2, 1):                      # release 1 MiB, 2 MiB, 1 MiB -> 4 MiB idle > 3 MiB cap
            a = hm.empty((mb << 20,), np.uint8)
            a[:] = 7
            del a
        assert hm.cached_bytes() <= 3 << 20
        assert hm.cached_bytes() == 3 << 20       # the OLDEST (first 1 MiB) block was evicted
        b = hm.empty((2 << 20,), np.uint8)        # recycled, no new allocation
        assert hm.cached_bytes() == 1 << 20
        del b
        big = hm.empty((4 << 20,), np.uint8)      # larger than the cap: freed on release, never cached
        del big
        assert hm.cached_bytes() <= 3 << 20
    finally:
        hm.MAX_CACHED_BYTES = old
        hm.trim()
    assert hm.cached_bytes() == 0


def test_host_path_over_several_devices_matches_one_device(xb, monkeypatch):
    """xrs_host_stencil over a list of devices: row stripes over the visible GPUs, halos from the host
    raster: the result is the single-device result bit for bit (with one GPU the stripes collapse to one)."""
    rng = np.random.default_rng(77)
    z = terrain(rng, 1500, 1024, nans=0.003)
    kern = rng.standard_normal((9, 9))
    n = torch.cuda.device_count()
    monkeypatch.setenv("XRS_B200_DEVICES", "0")
    one = {"slope": xb.slope(da(xb, z)).data.copy(), "mean": xb.mean(da(xb, z)).data.copy(),
           "conv": xb.convolve_2d(z, kern).copy(), "i16": xb.slope(da(xb, np.round(z).astype(np.int16))).data.copy()}
    monkeypatch.setenv("XRS_B200_DEVICES", "all")
    from xrspatial_b200 import utils
    assert utils.host_devices() == list(range(n))
    many = {"slope": xb.slope(da(xb, z)).data, "mean": xb.mean(da(xb, z)).data, "conv": xb.convolve_2d(z, kern),
            "i16": xb.slope(da(xb, np.round(z).astype(np.int16))).data}
    for k in one:
        np.testing.assert_array_equal(one[k], many[k], err_msg=k)
    assert_close_f32(many["slope"], o.slope(z, 30.0, 30.0), what="slope")
    monkeypatch.setenv("XRS_B200_DEVICES", "0,0")
    with pytest.raises(ValueError):
        xb.slope(da(xb, z))
    monkeypatch.setenv("LOCAL_RANK", "0")
    monkeypatch.delenv("XRS_B200_DEVICES")
    assert utils.host_devices() == [torch.cuda.current_device()]      # one process per GPU: own device only


def test_synthetic_dem_host_twin_matches_the_device_generator(xb):
    """oracle.synth_terrain (bench.py's CPU arms) == xrs_synth_terrain_f32 to float32 rounding, for an
    offset window -- the generator is a pure function of (seed, global row, global col)."""
    import ctypes
    t = torch.empty((300, 512), dtype=torch.float32, device="cuda")
    xb._lib.call("xrs_synth_terrain_f32", ctypes.c_void_p(t.data_ptr()), 512 * 4, 300, 512, 4100, 8192, 1235, 0.0, 4000.0,
                 ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    ref = o.synth_terrain(300, 512, 4100, 8192, 1235, 0.0, 4000.0, nthreads=4)
    np.testing.assert_allclose(t.cpu().numpy(), ref, rtol=2e-6, atol=2e-3)


def test_zonal_many_zones_and_degenerate_rasters(xb):
    """hash_partials: more zones than the one-copy fast path returns (4096) fall back to gathering the
    table; 1-cell and empty rasters; a zone whose cells are all invalid is still reported (NaN row)."""
    rng = np.random.default_rng(19)
    zones = rng.integers(0, 6000, size=(512, 640)).astype(np.int32)
    vals = rng.standard_normal((512, 640)).astype(np.float32) * 50 + 300
    vals[zones == 17] = np.nan
    cols = ["mean", "max", "min", "sum", "std", "var", "count"]
    df = xb.zonal_stats(da(xb, dev(zones)), da(xb, dev(vals)), stats_funcs=cols)
    ref = o.zonal_stats(zones, vals, stats_funcs=cols)
    assert len(df) == len(np.unique(zones)) > 4096
    np.testing.assert_array_equal(np.asarray(df["zone"]), ref["zone"])
    for c in ("count", "min", "max"):
        np.testing.assert_array_equal(np.asarray(df[c], dtype=np.float64), ref[c], err_msg=c)
    for c in ("mean", "sum", "std", "var"):
        np.testing.assert_allclose(np.asarray(df[c], dtype=np.float64), ref[c], rtol=1e-5, atol=1e-4, equal_nan=True, err_msg=c)
    row = df[df["zone"] == 17]
    assert len(row) == 1 and np.isnan(row["mean"].iloc[0]) and np.isnan(row["count"].iloc[0])
    one = xb.zonal_stats(da(xb, dev(np.array([[3]], np.int32))), da(xb, dev(np.array([[2.5]], np.float32))), stats_funcs=cols)
    assert list(one["zone"]) == [3] and one["mean"].iloc[0] == 2.5 and one["count"].iloc[0] == 1 and one["var"].iloc[0] == 0
    emp = xb.zonal_stats(da(xb, dev(np.zeros((0, 8), np.int32))), da(xb, dev(np.zeros((0, 8), np.float32))), stats_funcs=cols)
    assert len(emp) == 0 and list(emp.columns) == ["zone"] + cols


@pytest.mark.parametrize("k", [5, 9, 15, 25])
def test_streaming_box_convolve_many_tiles_and_sentinels(xb, k):
    """box_stream.cu on a raster spanning several CTA tiles and row segments, with scattered NaN, +-inf
    and a FLT_MAX-style nodata sentinel: windows holding a NaN are NaN, windows holding an infinite /
    huge cell come back in the reference's tap order, and every OTHER window is unaffected by a bad
    cell that passed through the running sums' neighbourhood (the round-1 summed-area table lost
    those: ADVICE r1)."""
    from xrspatial_b200.convolution import convolve_2d
    rng = np.random.default_rng(1000 + k)
    z = terrain(rng, 2100, 2304)
    kern = np.ones((k, k)) / (k * k)
    ref = o.convolve_2d(z, kern, nthreads=16)
    got = convolve_2d(dev(z), kern).cpu().numpy()
    assert used_tma(xb) == 3
    assert_close_f32(got, ref, atol=1e-6 * 4000.0, what="box %d clean" % k)
    d = z.copy()
    d[rng.random(d.shape) < 0.0005] = np.nan
    d[700, 1000] = np.inf
    d[1500, 40] = -np.inf
    d[300:305, 2000:2003] = np.float32(3.4028235e38)     # nodata sentinel: finite, huge
    d[1800, 1200] = np.float32(-3.4028235e38)
    d[40, 2303] = np.float32(1e31)
    ref = o.convolve_2d(d, kern, nthreads=16)
    got = convolve_2d(dev(d), kern).cpu().numpy()
    assert used_tma(xb) == 3
    fin = np.isfinite(ref) & (np.abs(ref) < 1e20)
    assert_close_f32(np.where(fin, got, 0), np.where(fin, ref, 0), atol=1e-6 * 4000.0, what="box %d, ordinary windows" % k)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
    big = ~np.isnan(ref) & ~fin
    assert big.any()
    np.testing.assert_allclose(got[big], ref[big], rtol=1e-6)         # same tap order: same inf / huge values
    # rectangular windows and a negative weight
    for kh, kw in ((k, 3), (3, k), (1, k)):
        kern2 = np.full((kh, kw), -0.25)
        ref = o.convolve_2d(z[:600], kern2, nthreads=16)
        got = convolve_2d(dev(z[:600]), kern2).cpu().numpy()
        assert used_tma(xb) == 3
        assert_close_f32(got, ref, atol=1e-6 * np.nanmax(np.abs(ref)), what="box %dx%d" % (kh, kw))


@pytest.mark.parametrize("kh,kw", [(5, 5), (25, 25), (3, 7), (9, 3), (1, 5), (15, 15)])
def test_focal_apply_mean_over_all_ones_windows_takes_the_running_box(xb, kh, kw):
    """focal.apply(raster, np.ones((kh, kw))) -- the reference's own focal benchmark (benchmarks/focal.py
    FocalApply) -- runs on the running-box kernel in NaN-skipping mode: NaN cells and cells beyond the raster
    are skipped (clamped windows at the edges), infinite cells take part, an all-NaN window is NaN
    (focal.py:268-270, 305-326)."""
    from xrspatial_b200 import focal
    rng = np.random.default_rng(7000 + 31 * kh + kw)
    z = terrain(rng, 1300, 2052)                      # several CTA tiles and row segments
    kern = np.ones((kh, kw))
    got = host(focal.apply(da(xb, dev(z)), kern))
    assert used_tma(xb) == 3
    assert_close_f32(got, o.focal_apply(z, kern, "mean", nthreads=16), what="apply mean %dx%d clean" % (kh, kw))
    d = z.copy()
    d[rng.random(d.shape) < 0.002] = np.nan
    d[200:240, 300:340] = np.nan                      # all-NaN windows (for the smaller kernels)
    d[700, 1000] = np.inf
    d[900, 40] = -np.inf
    d[1100:1103, 2000:2003] = np.float32(3.4028235e38)
    ref = o.focal_apply(d, kern, "mean", nthreads=16)
    got = host(focal.apply(da(xb, dev(d)), kern))
    assert used_tma(xb) == 3
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
    fin = np.isfinite(ref) & (np.abs(ref) < 1e20)
    assert_close_f32(np.where(fin, got, 0), np.where(fin, ref, 0), what="apply mean %dx%d, ordinary windows" % (kh, kw))
    odd = ~np.isnan(ref) & ~fin
    assert odd.any()
    np.testing.assert_allclose(got[odd], ref[odd], rtol=1e-6)      # infinite / huge windows: the reference's order
    # the other reducers keep the tiled kernel
    sub = d[:260, :512]
    assert_close_f32(host(focal.apply(da(xb, dev(sub)), kern, func="max")), o.focal_apply(sub, kern, "max", nthreads=8),
                     what="apply max %dx%d" % (kh, kw))


def test_crosstab_3d(xb, known, refout):
    """zonal.py:1096-1116 / :734-745: 3-D `values`, categories = coordinate of dimension `layer`, cell =
    statistic `agg` of the layer over the zone.  The reference's own fixtures (test_zonal.py:48-58,
    266-336) and its per-zone loop on a seeded raster."""
    zones = known["zonal.data_zones"]
    v3 = np.ones(4 * 3 * 8).reshape(3, 8, 4)
    layer = int(known["zonal.result_crosstab_3d.layer"])
    for mk in (dev, lambda a: a):
        zagg = xb.DataArray(mk(zones), dims=("lat", "lon"))
        vagg = xb.DataArray(mk(v3), dims=("lat", "lon", "race"))
        vagg["race"] = ["cat1", "cat2", "cat3", "cat4"]
        for agg in ("min", "max", "mean", "sum", "std", "var", "count"):
            df = xb.zonal_crosstab(zagg, vagg, zone_ids=[1, 2, 3], layer=layer, agg=agg)
            assert list(df.columns) == ["zone", "cat1", "cat2", "cat3", "cat4"]
            np.testing.assert_allclose(np.asarray(df.values, dtype=np.float64).T, known["zonal.result_crosstab_3d." + agg],
                                       rtol=1e-6, atol=1e-7, err_msg=agg)
        df = xb.zonal_crosstab(zagg, vagg, zone_ids=[1, 2, 3], layer=layer, nodata_values=1)
        np.testing.assert_array_equal(np.asarray(df.values, dtype=np.float64).T, known["zonal.result_nodata_values_crosstab_3d"])
        with pytest.raises(ValueError, match="Invalid `layer`"):
            xb.zonal_crosstab(zagg, vagg, layer=0)            # 'lat' carries no coordinate
        with pytest.raises(ValueError, match="Incompatible shapes"):
            xb.zonal_crosstab(xb.DataArray(mk(zones[:, :5]), dims=("lat", "lon")), vagg, layer=layer)
    r = refout
    cz, c3 = r["crosstab.zones"], r["crosstab3d.values"]
    vagg = xb.DataArray(dev(c3), dims=("year", "y", "x"))
    vagg["year"] = [2001.0, 2002.0, 2003.0, 2004.0]
    zagg = xb.DataArray(dev(cz), dims=("y", "x"))
    for agg in ("mean", "max", "min", "sum", "std", "var", "count"):
        df = xb.zonal_crosstab(zagg, vagg, zone_ids=[0, 1, 2, 3, 5], cat_ids=[2001.0, 2003.0, 2004.0], nodata_values=7.0,
                               agg=agg)
        assert list(df.columns) == ["zone", 2001.0, 2003.0, 2004.0]
        np.testing.assert_allclose(np.asarray(df.values, dtype=np.float64), r["crosstab3d." + agg], rtol=1e-5, atol=1e-4,
                                   err_msg=agg)


def test_running_box_every_radius(xb):
    """The running box at every window width 5..25 (every compile-time radius: each has its own shuffle
    pattern), square and 3-row windows, against the oracle: clean raster, then NaN / inf / sentinel cells
    including ones next to the raster's edges (a window that holds an infinite cell AND reaches beyond the raster
    is NaN, not the tap-order recompute).  The same loop run on the CPU through the NumPy statement of the
    algorithm (tests/test_kernel_algebra.py `_box_running`) meets these expectations at every width."""
    from xrspatial_b200 import focal
    from xrspatial_b200.convolution import convolve_2d
    rng = np.random.default_rng(4242)
    z = terrain(rng, 150, 2052)
    d = z.copy()
    d[rng.random(d.shape) < 0.001] = np.nan
    d[40, 2] = np.inf                    # within every radius >= 2 of the left edge
    d[90, 2049] = np.float32(3.4028235e38)
    d[100, 1000] = -np.inf
    d[3, 500] = np.inf                   # near the top edge
    for kw in range(5, 26, 2):
        for kh in sorted({kw, 3}):
            kern = np.full((kh, kw), 1.0 / (kh * kw))
            for data in (z, d):
                ref = o.convolve_2d(data, kern, nthreads=16)
                got = convolve_2d(dev(data), kern).cpu().numpy()
                assert used_tma(xb) == 3
                np.testing.assert_array_equal(np.isnan(got), np.isnan(ref), err_msg="NaN mask %dx%d" % (kh, kw))
                fin = np.isfinite(ref) & (np.abs(ref) < 1e20)
                assert_close_f32(np.where(fin, got, 0), np.where(fin, ref, 0), atol=1e-6 * 4000.0, what="box %dx%d" % (kh, kw))
                odd = ~np.isnan(ref) & ~fin
                np.testing.assert_allclose(got[odd], ref[odd], rtol=1e-6)
        if kw in (7, 11, 17, 19, 21, 23):
            kern = np.ones((kw, kw))
            ref = o.focal_apply(d, kern, "mean", nthreads=16)
            got = host(focal.apply(da(xb, dev(d)), kern))
            assert used_tma(xb) == 3
            np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
            fin = np.isfinite(ref) & (np.abs(ref) < 1e20)
            assert_close_f32(np.where(fin, got, 0), np.where(fin, ref, 0), what="apply mean %dx%d" % (kw, kw))
            odd = ~np.isnan(ref) & ~fin
            np.testing.assert_allclose(got[odd], ref[odd], rtol=1e-6)

"""convolve_2d and the focal statistics over windows beyond the tiled kernels: more than 49 x 49 taps or more
than 63 cells on a side, up to 2047 x 2047.

conv2d_wide_kernel must agree bit for bit with the FMA oracle (row-major fma(w, (double)x, acc) from +0.0 over
every tap, out-of-raster taps NaN), and focal_wide_kernel with the oracle's Numba reducers for mean, sum, min,
max and range (var and std within the bound of test_kxk_edges).  The fused kernel's planes
(focal_wide_kernel<kAllStats>) must equal the single-statistic calls bit for bit.  The harness is test_kxk_edges's: the input inside a buffer of large
finite cells, the output inside a sentinel-filled pitched buffer, and an assert on the kernel that ran.  The
oracle is O(taps) per cell, so the large windows run on small rasters.  Runs on an H100 (`-m gpu`)."""
import ctypes

import numpy as np
import pytest

import oracle as o
from helpers import Pitched, in_buffer, raster, stream, terrain
from test_kxk_edges import (EXACT_STATS, STATS, _bits_equal, _circle, _launch, _mixed, _signed_zero_raster,
                            _var_bound)

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

K_CONV_WIDE, K_STAT_WIDE, K_FUSED_WIDE = 11, 12, 13   # LaunchKind in csrc/common.cuh


@pytest.fixture(scope="module")
def lib():
    from helpers import gpu_lib
    return gpu_lib()


def _conv(lib, z, k, view, what):
    H, W = z.shape
    kk = np.ascontiguousarray(k, dtype=np.float64)
    return _launch(lib, lambda i, ip, out, op: lib.call("xrs_convolve2d_f32", i, ip, out, op, H, W, kk.ctypes.data,
                                                         k.shape[0], k.shape[1], stream()),
                   z, view, K_CONV_WIDE, what)


def _check_conv(lib, z, k, what, views=({},)):
    ref = o.convolve_2d_fma(z, k, nthreads=o.max_threads())
    for view in views:
        _bits_equal(_conv(lib, z, k, view, "%s %s" % (what, view)), ref, "%s %s: vs FMA oracle" % (what, view))


# ------------------------------------------------------------------------------------------------ convolve_2d
WIDE_SHAPES = [(49, 51), (51, 51), (65, 1), (1, 65), (257, 1), (1, 257), (101, 101), (75, 131)]


@pytest.mark.parametrize("kh,kw", WIDE_SHAPES)
def test_convolve_heights(lib, kh, kw):
    """Heights around the 4-row tile and around the window height."""
    k = _mixed(kh, kw, kh * 1000 + kw)
    for H in sorted({1, 2, 3, 4, 5, 8, kh - 1, kh, kh + 1} - {0}):
        _check_conv(lib, raster(H, 132, H + kh), k, "%dx%d on %dx132" % (kh, kw, H))


@pytest.mark.parametrize("kh,kw", WIDE_SHAPES)
def test_convolve_widths(lib, kh, kw):
    """Widths around the 128-cell groups, the 2048-cell tile, and W % 4 != 0."""
    k = _mixed(kh, kw, kh + kw)
    for W in (4, 124, 128, 132, 260, 2052, 1030):
        _check_conv(lib, raster(7, W, W + kh), k, "%dx%d on 7x%d" % (kh, kw, W))


def test_convolve_very_wide_windows(lib):
    _check_conv(lib, raster(70, 140, 1), _mixed(201, 201, 2), "201x201 on 70x140")
    _check_conv(lib, raster(9, 21, 3), _mixed(2047, 2047, 4), "2047x2047 on 9x21")
    _check_conv(lib, raster(5, 2100, 5), _mixed(3, 2047, 6), "3x2047 on 5x2100")


def test_convolve_zero_taps(lib):
    """Circle weights x 0.01: a NaN or inf under a zero tap still makes the window NaN."""
    for k in (101, 67):
        w = _circle(k) * 0.01
        w[k // 2, k // 2] = -0.5
        z = raster(90, 260, k, nan_frac=0.001)
        rng = np.random.default_rng(k)
        z[rng.random(z.shape) < 0.0005] = np.inf
        z[rng.random(z.shape) < 0.0005] = -np.inf
        _check_conv(lib, z, w, "circle %d" % k)


@pytest.mark.parametrize("kh,kw", [(51, 51), (1, 257), (101, 65)])
def test_convolve_pitched_offset_and_shifted_views(lib, kh, kw):
    k = _mixed(kh, kw, 7 * kh + kw)
    for W in (252, 2052, 130):
        pad = (-(W * 4) % 128 + 16) // 4
        z = raster(37, W, W)
        _check_conv(lib, z, k, "%dx%d W %d" % (kh, kw, W),
                    views=({"pad_cols": pad}, {"rows_above": 3, "rows_below": 2}, {"shift": 1}))


def test_convolve_window_larger_than_raster(lib):
    for kh, kw, H, W in ((201, 201, 30, 40), (101, 101, 1, 1), (65, 65, 1, 300), (1, 301, 1, 7), (301, 1, 5, 1)):
        _check_conv(lib, raster(H, W, kh + H + W), _mixed(kh, kw, W), "%dx%d on %dx%d" % (kh, kw, H, W),
                    views=({}, {"shift": 1}))


# ----------------------------------------------------------------------------------------- focal statistics
def _stat(lib, z, k, stat, view, what):
    H, W = z.shape
    kk = np.ascontiguousarray(k, dtype=np.float64)
    return _launch(lib, lambda i, ip, out, op: lib.call("xrs_focal_stat_f32", i, ip, out, op, H, W, kk.ctypes.data,
                                                         k.shape[0], k.shape[1], STATS[stat], stream()),
                   z, view, K_STAT_WIDE, "%s %s" % (stat, what))


def _check_stats(lib, z, k, what, view={}):
    for stat in STATS:
        got = _stat(lib, z, k, stat, view, what)
        orc = o.focal_apply(z, k, stat, nthreads=o.max_threads())
        if stat in EXACT_STATS:
            _bits_equal(got, orc, "%s %s: vs oracle" % (stat, what))
        else:
            _var_bound(got, orc, k, "%s %s" % (stat, what))


def _wide_masks():
    ann = _circle(101) - _circle(101, 20)
    first_row_zero = np.ones((55, 55))
    first_row_zero[0] = 0
    odd_values = _circle(65)
    odd_values[1, 32] = 0.5
    odd_values[32, 1] = 2.0
    odd_values[40, 40] = 0.5
    return {"circle51": _circle(51), "circle101": _circle(101), "circle201": _circle(201), "annulus101_41": ann,
            "rect3x129": np.ones((3, 129)), "rect129x3": np.ones((129, 3)), "ones51": np.ones((51, 51)),
            "first_row_zero": first_row_zero, "values_0.5_2": odd_values}


@pytest.mark.parametrize("name", list(_wide_masks()))
def test_focal_stats_masks(lib, name):
    k = _wide_masks()[name]
    big = k.shape[0] * k.shape[1] > 20000                           # small rasters for the oracle
    for H, W in (((40, 132), (9, 260)) if big else ((70, 260), (9, 132), (3, 1030))):
        _check_stats(lib, raster(H, W, H + W + k.size), k, "%s on %dx%d" % (name, H, W))
        z = _signed_zero_raster(H, W, H * W)
        z[H // 2:, W // 2:] = np.nan                                     # all-NaN windows
        _check_stats(lib, z, k, "%s signed zeros on %dx%d" % (name, H, W))


def test_focal_stats_views(lib):
    k = _wide_masks()["annulus101_41"]
    for W in (252, 130):
        pad = (-(W * 4) % 128 + 16) // 4
        z = _signed_zero_raster(23, W, W)
        for view in ({"pad_cols": pad}, {"rows_above": 3, "rows_below": 2}, {"shift": 1}):
            _check_stats(lib, z, k, "W %d %s" % (W, view), view)


def test_min_max_keep_the_last_of_equal_zeros(lib):
    z = np.ones((8, 132), np.float32)
    z[3, 20], z[3, 21] = np.float32(-0.0), np.float32(0.0)
    z[5, 60], z[5, 61] = np.float32(0.0), np.float32(-0.0)
    k = np.ones((1, 65))
    k[0, 33:] = 0                                                        # the window ends at the centre + 0
    for stat in ("min", "max", "range"):
        _bits_equal(_stat(lib, z, k, stat, {}, "zeros"), o.focal_apply(z, k, stat), "%s vs oracle" % stat)


def _fused(lib, z, k, stats, kind=K_FUSED_WIDE):
    H, W = z.shape
    kk = np.ascontiguousarray(k, dtype=np.float64)
    ids = np.array([STATS[s] for s in stats], dtype=np.int32)
    t, ptr, pitch = in_buffer(z)
    plane = (H * W * 4 + 15) // 16 * 16
    out = torch.full((len(ids) * plane // 4,), -1.0, dtype=torch.float32, device="cuda")
    lib.call("xrs_focal_stats_multi_f32", ptr, pitch, out.data_ptr(), W * 4, plane, H, W, kk.ctypes.data,
             k.shape[0], k.shape[1], ids.ctypes.data, len(ids), stream())
    torch.cuda.synchronize()
    assert lib.lib().xrs_debug_last_used_tma() == kind
    res = out.cpu().numpy()
    return {s: res[i * plane // 4:i * plane // 4 + H * W].reshape(H, W) for i, s in enumerate(stats)}


@pytest.mark.parametrize("name", ["circle51", "annulus101_41", "first_row_zero"])
def test_fused_planes_equal_single_calls(lib, name):
    """2 to 7 statistics in shuffled orders: every plane bit-identical to xrs_focal_stat_f32."""
    k = _wide_masks()[name]
    rng = np.random.default_rng(len(name))
    for H, W in ((41, 260), (6, 130)):
        z = _signed_zero_raster(H, W, H + W)
        single = {s: _stat(lib, z, k, s, {}, "single") for s in STATS}
        for n in range(2, 8):
            stats = list(rng.permutation(list(STATS))[:n])
            for s, got in _fused(lib, z, k, stats).items():
                _bits_equal(got, single[s], "fused %s of %s, %s %dx%d" % (s, stats, name, H, W))


def test_two_streams(lib):
    """Wide convolves and wide focal maxima enqueued on two streams, alternating, with no synchronisation until all
    eight are in flight: each call's weight / mask table lives on its own stream."""
    s = [torch.cuda.Stream(), torch.cuda.Stream()]
    jobs = []
    for i in range(4):
        z1, z2 = raster(100, 1030, i), _signed_zero_raster(150, 516, i)
        k1, k2 = _mixed(101, 101, i), _circle(75)
        k2[37, 37] = 0.0 if i % 2 else 1.0                      # the two masks differ
        (t1, p1, pitch1), (t2, p2, pitch2) = in_buffer(z1), in_buffer(z2)
        o1, o2 = Pitched(*z1.shape), Pitched(*z2.shape)
        jobs.append((z1, k1, t1, p1, pitch1, o1, z2, k2, t2, p2, pitch2, o2))
    torch.cuda.synchronize()
    for i, (z1, k1, t1, p1, pitch1, o1, z2, k2, t2, p2, pitch2, o2) in enumerate(jobs):
        lib.call("xrs_convolve2d_f32", p1, pitch1, o1.ptr, o1.pitch, 100, 1030, k1.ctypes.data, 101, 101,
                 ctypes.c_void_p(s[i % 2].cuda_stream))
        assert lib.lib().xrs_debug_last_used_tma() == K_CONV_WIDE
        lib.call("xrs_focal_stat_f32", p2, pitch2, o2.ptr, o2.pitch, 150, 516, k2.ctypes.data, 75, 75,
                 STATS["max"], ctypes.c_void_p(s[1 - i % 2].cuda_stream))
        assert lib.lib().xrs_debug_last_used_tma() == K_STAT_WIDE
    torch.cuda.synchronize()
    for i, (z1, k1, t1, p1, pitch1, o1, z2, k2, t2, p2, pitch2, o2) in enumerate(jobs):
        _bits_equal(o1.inside("convolve %d" % i).view(np.float32),
                    o.convolve_2d_fma(z1, k1, nthreads=o.max_threads()), "convolve %d" % i)
        _bits_equal(o2.inside("max %d" % i).view(np.float32),
                    o.focal_apply(z2, k2, "max", nthreads=o.max_threads()), "max %d" % i)


def test_host_path_at_radius_1023(xb):
    """Numpy rasters through xrs_host_stencil with a 2047-row window: chunks of at least 8r + 8 = 8192 rows, capped
    at the raster, and halos larger than the raster."""
    from xrspatial_b200 import focal
    from xrspatial_b200.convolution import convolution_2d
    z = raster(300, 40, 11)
    agg = xb.DataArray(z, dims=("y", "x"), attrs={"res": (1, 1)})
    k = _mixed(2047, 3, 12)
    got = np.asarray(convolution_2d(agg, k).data)
    _bits_equal(got, o.convolve_2d_fma(z, k, nthreads=o.max_threads()), "host convolve 2047x3")
    m = np.ones((2047, 1))
    m[::3] = 0
    for stat in ("mean", "max"):
        got = np.asarray(focal.apply(agg, m, func=stat).data)
        _bits_equal(got, o.focal_apply(z, m, stat, nthreads=o.max_threads()), "host %s 2047x1" % stat)


# ------------------------------------------------------------------------------------------------ public API
@pytest.fixture(scope="module")
def xb():
    import xrspatial_b200
    return xrspatial_b200


def _both(xb, fn, z):
    """fn on a device raster and on a numpy raster: identical results; returns the host array."""
    dev = fn(xb.DataArray(torch.from_numpy(z).cuda(), dims=("y", "x"), attrs={"res": (1, 1)})).data.cpu().numpy()
    host = np.asarray(fn(xb.DataArray(z, dims=("y", "x"), attrs={"res": (1, 1)})).data)
    np.testing.assert_array_equal(dev.view(np.uint8), host.view(np.uint8))
    return host


def test_public_api_wide_kernels(xb):
    from xrspatial_b200 import focal
    from xrspatial_b200.convolution import annulus_kernel, circle_kernel, convolution_2d
    z = terrain(np.random.default_rng(5), 150, 260, nans=0.01)
    circle, ann = circle_kernel(1, 1, 30), annulus_kernel(1, 1, 60, 20)
    assert circle.shape == (61, 61) and ann.shape == (121, 121)
    for k in (circle, ann):
        got = _both(xb, lambda a: convolution_2d(a, k), z)
        _bits_equal(got, o.convolve_2d_fma(z, k, nthreads=o.max_threads()), "convolution_2d %s" % (k.shape,))
        for stat in ("mean", "max", "sum"):
            got = _both(xb, lambda a: focal.apply(a, k, func=stat), z)
            _bits_equal(got, o.focal_apply(z, k, stat, nthreads=o.max_threads()), "apply %s %s" % (stat, k.shape))
        stats = list(STATS)
        got = _both(xb, lambda a: focal.focal_stats(a, k, stats_funcs=stats), z)
        for i, stat in enumerate(stats):
            orc = o.focal_apply(z, k, stat, nthreads=o.max_threads())
            if stat in EXACT_STATS:
                _bits_equal(got[i], orc, "focal_stats %s %s" % (stat, k.shape))
            else:
                _var_bound(got[i], orc, k, "focal_stats %s %s" % (stat, k.shape))


def test_public_api_hotspots(xb):
    from xrspatial_b200.convolution import circle_kernel
    z = terrain(np.random.default_rng(9), 180, 300, nans=0.01)
    k = circle_kernel(1, 1, 30)
    got = _both(xb, lambda a: xb.hotspots(a, k), z)
    mean = o.convolve_2d_fma(z, k / k.sum(), nthreads=o.max_threads())
    d = z.astype(np.float64)
    zs = (mean - np.float32(np.nanmean(d))) / np.float32(np.nanstd(d))
    az = np.abs(zs.astype(np.float64))
    cls = np.where(az > 2.58, 99, np.where(az > 1.96, 95, np.where(az > 1.65, 90, 0))) * np.sign(zs)
    cls = np.where(np.isnan(zs), 0, cls).astype(np.int8)
    far = np.ones(z.shape, bool)
    for b in (1.29, 1.65, 1.96, 2.33, 2.58):
        far &= ~(np.abs(az - b) <= 1e-4)
    assert far.sum() > 0.9 * z.size
    np.testing.assert_array_equal(got[far], cls[far])


def test_public_api_rejects_sides_above_2047(xb):
    from xrspatial_b200 import focal
    from xrspatial_b200.convolution import convolution_2d
    z = np.zeros((6, 8), np.float32)
    for data in (z, torch.from_numpy(z).cuda()):
        agg = xb.DataArray(data, dims=("y", "x"), attrs={"res": (1, 1)})
        for k in (np.ones((2049, 1)), np.ones((1, 2049))):
            for call in (lambda: convolution_2d(agg, k), lambda: focal.apply(agg, k),
                         lambda: focal.focal_stats(agg, k, stats_funcs=["mean", "max"]),
                         lambda: xb.hotspots(agg, k)):
                with pytest.raises(ValueError):
                    call()

"""The k x k convolution and focal-statistics kernels at their tile, halo and magnitude edges.

conv2d_kernel / conv2d_fixed_kernel (128 x 64 output tiles), the 3 x 3 strip kernels and conv2d_direct_kernel all
compute acc = fma(w, (double)x, acc) in row-major tap order from +0.0 with out-of-raster cells NaN, so they must
agree bit for bit with each other and with the FMA oracle (oracle.convolve_2d_fma).  focal_stat_kernel (128 x 32
tiles) and focal_stat_direct_kernel share Numba's nan-reducers, so mean, sum, min, max and range must agree bit
for bit, sign bits included.  The running box (uniform convolve_2d and focal.apply mean over all-ones windows) is
held to a per-window bound at planted magnitudes from 2^24 M to FLT_MAX.

Every case calls the C entry points with the input inside a larger buffer of large finite cells (a read outside
the raster shows up) and the output inside a sentinel-filled pitched buffer (a write outside H x W shows up), and
asserts which kernel ran.  Runs on an H100 (`-m gpu`)."""
import ctypes

import numpy as np
import pytest

import oracle as o
from helpers import box_magnitude_fields, box_plant, box_planted_values, box_window_errors

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

SENTINEL = 0x5A
STATS = {"mean": 0, "sum": 1, "min": 2, "max": 3, "std": 4, "range": 5, "var": 6}
EXACT_STATS = ("mean", "sum", "min", "max", "range")
# launch codes of xrs_debug_last_used_tma
K_STRIP_CPASYNC, K_STRIP_TMA, K_BOX, K_CONV_TILED, K_CONV_DIRECT, K_FUSED, K_STAT_TILED, K_STAT_DIRECT = \
    0, 1, 3, 4, 5, 6, 7, 8
WIDTHS = [4, 124, 128, 132, 252, 256, 260, 2044, 2052]


@pytest.fixture(scope="module")
def lib():
    import xrspatial_b200
    assert torch.cuda.is_available(), "these tests need a CUDA device"
    return xrspatial_b200._lib


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _heights(kh):
    return sorted({h for h in (1, 2, kh - 1, kh, kh + 1, 63, 64, 65, 129) if h >= 1})


def _raster(H, W, seed, nan_frac=0.01):
    rng = np.random.default_rng(seed)
    z = rng.standard_normal((H, W)).cumsum(0).cumsum(1) * 3.0 + 500.0
    z[rng.random((H, W)) < nan_frac] = np.nan
    return z.astype(np.float32)


def _in_buffer(z, pad_cols=0, rows_above=0, rows_below=0, shift=0):
    """z on the device inside a larger buffer: `pad_cols` extra cells per row (pitch), `rows_above` /
    `rows_below` extra rows (a row-offset view), `shift` cells past the 16-byte aligned start (no TMA: the
    bounds-checked kernels).  The extra cells hold a large finite value."""
    H, W = z.shape
    big = np.full((H + rows_above + rows_below, W + pad_cols + shift), 9.0e3, dtype=np.float32)
    big[rows_above:rows_above + H, shift:shift + W] = z
    t = torch.from_numpy(big).cuda()
    return t, t.data_ptr() + (rows_above * t.stride(0) + shift) * 4, t.stride(0) * 4


class Pitched(object):
    """An H x W float32 output inside a sentinel-filled buffer: one row above and below, 4 cells left and 8
    right (pitch a multiple of 16 bytes)."""

    def __init__(self, H, W):
        self.H, self.W = H, W
        self.wp = W + 12
        self.buf = torch.full(((H + 2) * self.wp * 4,), SENTINEL, dtype=torch.uint8, device="cuda")
        self.ptr = self.buf.data_ptr() + (self.wp + 4) * 4
        self.pitch = self.wp * 4

    def inside(self, what):
        b = self.buf.cpu().numpy().reshape(self.H + 2, self.pitch)
        ins = b[1:1 + self.H, 16:16 + 4 * self.W].copy()
        b[1:1 + self.H, 16:16 + 4 * self.W] = SENTINEL
        bad = int((b != SENTINEL).sum())
        assert bad == 0, "%s: %d bytes outside the raster were written" % (what, bad)
        return ins.view(np.float32).reshape(self.H, self.W)


def _launch(lib, call, z, view, kind, what):
    """Run `call(in_ptr, in_pitch, out_ptr, out_pitch)` on z placed as `view`; check the kernel and the
    untouched border; return the float32 result."""
    H, W = z.shape
    t, ptr, pitch = _in_buffer(z, **view)
    out = Pitched(H, W)
    call(ptr, pitch, out.ptr, out.pitch)
    torch.cuda.synchronize()
    got_kind = lib.lib().xrs_debug_last_used_tma()
    assert got_kind == kind, "%s: kernel %d ran, expected %d" % (what, got_kind, kind)
    return out.inside(what)


def _bits_equal(a, b, what):
    """Same NaN mask and, everywhere else, the same bits (sign of zero included).  A NaN's sign and payload
    depend on which operand the hardware propagates and carry no meaning, so they are not compared."""
    np.testing.assert_array_equal(np.isnan(a), np.isnan(b), err_msg=what + ": NaN masks differ")
    a32 = np.where(np.isnan(a), np.float32(np.nan), a).view(np.uint32)
    b32 = np.where(np.isnan(b), np.float32(np.nan), b).view(np.uint32)
    bad = a32 != b32
    if bad.any():
        i = np.argwhere(bad)[0]
        raise AssertionError("%s: %d cells differ in their bits, first at %s: %r vs %r"
                             % (what, int(bad.sum()), tuple(i), a[tuple(i)], b[tuple(i)]))


# ------------------------------------------------------------------------------------------------ convolve_2d
def _conv_call(lib, k):
    kh, kw = k.shape
    kk = np.ascontiguousarray(k, dtype=np.float64)

    def call(i, ip, out, op, H, W):
        lib.call("xrs_convolve2d_f32", i, ip, out, op, H, W, kk.ctypes.data, kh, kw, _stream())
    return call


def _tiled_kind(k):
    kh, kw = k.shape
    return (K_STRIP_TMA if kh == kw == 3 else K_CONV_TILED)


def _check_conv(lib, z, k, view, what, oracle_too=True):
    H, W = z.shape
    call = _conv_call(lib, k)
    kind = _tiled_kind(k)
    got = _launch(lib, lambda i, ip, out, op: call(i, ip, out, op, H, W), z, view,
                  kind if W % 4 == 0 else (K_STRIP_CPASYNC if k.shape == (3, 3) else K_CONV_DIRECT), what)
    ref = _launch(lib, lambda i, ip, out, op: call(i, ip, out, op, H, W), z, {"shift": 1},
                  K_STRIP_CPASYNC if k.shape == (3, 3) else K_CONV_DIRECT, what + " (direct)")
    _bits_equal(got, ref, what + ": tiled vs bounds-checked")
    if oracle_too:
        _bits_equal(got, o.convolve_2d_fma(z, k, nthreads=o.max_threads()), what + ": vs FMA oracle")


def _mixed(kh, kw, seed):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((kh, kw)) * 0.3


def _circle(k, r=None):
    r = k // 2 if r is None else r
    y, x = np.mgrid[:k, :k] - k // 2
    return (x * x + y * y <= r * r).astype(np.float64)


CONV_KERNELS = [(3, 3), (5, 5), (7, 7), (9, 9), (11, 11), (13, 13), (15, 15), (25, 25),
                (3, 5), (5, 9), (9, 5), (7, 1), (1, 31), (31, 1), (63, 1), (49, 49)]


@pytest.mark.parametrize("kh,kw", CONV_KERNELS)
def test_convolve_heights(lib, kh, kw):
    """Every height around the 64-row tile and the window height, at two widths around the 128-cell tile."""
    k = _mixed(kh, kw, kh * 100 + kw)
    for H in _heights(kh):
        for W in (132, 260):
            _check_conv(lib, _raster(H, W, H * 7 + W + kh), k, {}, "%dx%d on %dx%d" % (kh, kw, H, W),
                        oracle_too=kh * kw * H * W <= 3e7)


@pytest.mark.parametrize("kh,kw", CONV_KERNELS)
def test_convolve_widths(lib, kh, kw):
    """Every width around one and two 128-cell tiles and the 256-cell TMA box limit, including W = 4."""
    k = _mixed(kh, kw, kh * 10 + kw)
    for W in WIDTHS:
        H = 65
        _check_conv(lib, _raster(H, W, W + kh), k, {}, "%dx%d on %dx%d" % (kh, kw, H, W),
                    oracle_too=kh * kw * H * W <= 3e7)


@pytest.mark.parametrize("k", [5, 9, 25, 49])
def test_convolve_zero_taps(lib, k):
    """Circle weights: a NaN under a zero tap still makes the window NaN (0 * NaN is NaN in the reference)."""
    w = _circle(k) * 0.01
    w[k // 2, k // 2] = -0.5
    z = _raster(129, 260, k, nan_frac=0.003)
    _check_conv(lib, z, w, {}, "circle %d" % k)


@pytest.mark.parametrize("kh,kw", [(5, 5), (9, 5), (25, 25), (1, 31)])
def test_convolve_pitched_and_offset_views(lib, kh, kw):
    """A pitch that is a multiple of 16 B but not of 128 B, and a row-offset view whose neighbouring rows are
    other data (never read as the view's neighbours)."""
    k = _mixed(kh, kw, kh + kw)
    for W in (252, 2052):
        pad = (-(W * 4) % 128 + 16) // 4
        _check_conv(lib, _raster(67, W, W), k, {"pad_cols": pad}, "%dx%d pitch +16 B, W %d" % (kh, kw, W))
        _check_conv(lib, _raster(41, W, W + 1), k, {"rows_above": 3, "rows_below": 2},
                    "%dx%d row-offset view, W %d" % (kh, kw, W))


def test_convolve_kernel_larger_than_raster(lib):
    for kh, kw, H, W in ((25, 25, 7, 12), (49, 49, 20, 4), (63, 1, 30, 8), (1, 31, 3, 16)):
        _check_conv(lib, _raster(H, W, kh + H), _mixed(kh, kw, W), {}, "%dx%d on %dx%d" % (kh, kw, H, W))


# ----------------------------------------------------------------------------------------- focal statistics
def _stat_call(lib, k, stat):
    kh, kw = k.shape
    kk = np.ascontiguousarray(k, dtype=np.float64)

    def call(i, ip, out, op, H, W):
        lib.call("xrs_focal_stat_f32", i, ip, out, op, H, W, kk.ctypes.data, kh, kw, STATS[stat], _stream())
    return call


def _var_bound(got, ref, k, what):
    """var / std: within ulp32(ref) + 4 n 2^-53 var (std: ... + 4 n 2^-53 std), n = the window's taps."""
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref), err_msg=what + ": NaN masks differ")
    m = np.isfinite(ref)
    n = int((k == 1).sum())
    r = ref[m].astype(np.float64)
    bound = np.spacing(np.abs(ref[m])).astype(np.float64) + 4 * n * 2.0 ** -53 * np.abs(r)
    err = np.abs(got[m].astype(np.float64) - r)
    assert (err <= bound).all(), "%s: worst error %.3g over the bound" % (what, (err / bound).max())
    np.testing.assert_array_equal(got[~m & ~np.isnan(ref)], ref[~m & ~np.isnan(ref)])


def _check_stats(lib, z, k, view, what, stats=tuple(STATS)):
    H, W = z.shape
    for stat in stats:
        call = _stat_call(lib, k, stat)
        tiled = K_BOX if (stat == "mean" and (k == 1).all() and max(k.shape) <= 25 and k.shape[1] >= 3) \
            else K_STAT_TILED
        got = _launch(lib, lambda i, ip, out, op: call(i, ip, out, op, H, W), z, view,
                      tiled if W % 4 == 0 else K_STAT_DIRECT, "%s %s" % (stat, what))
        ref = _launch(lib, lambda i, ip, out, op: call(i, ip, out, op, H, W), z, {"shift": 1}, K_STAT_DIRECT,
                      "%s %s (direct)" % (stat, what))
        orc = o.focal_apply(z, k, stat, nthreads=o.max_threads())
        if tiled == K_BOX:     # running sums: the bound of the running-box tests
            M = float(np.abs(z[np.isfinite(z)]).max())
            box_window_errors(got, orc, np.zeros(z.shape, bool), k.shape[0], k.shape[1], 1.0, M,
                              "%s %s: running box vs oracle" % (stat, what))
            _bits_equal(ref, orc, "%s %s: bounds-checked vs oracle" % (stat, what))
        elif stat in EXACT_STATS:
            _bits_equal(got, ref, "%s %s: tiled vs bounds-checked" % (stat, what))
            _bits_equal(ref, orc, "%s %s: bounds-checked vs oracle" % (stat, what))
        else:
            _var_bound(got, orc, k, "%s %s tiled" % (stat, what))
            _var_bound(ref, orc, k, "%s %s bounds-checked" % (stat, what))


def _signed_zero_raster(H, W, seed):
    """Data with +0.0 / -0.0 pairs in both orders, NaN blocks (all-NaN windows, and windows whose only
    non-NaN cells are beyond the raster: none), +-inf, and 1e6 +- 0.01 offsets."""
    rng = np.random.default_rng(seed)
    z = (1e6 + np.round(rng.standard_normal((H, W)) * 100.0) * 0.01).astype(np.float32)
    zeros = rng.random((H, W)) < 0.25
    z[zeros] = np.where(rng.random(int(zeros.sum())) < 0.5, np.float32(0.0), np.float32(-0.0))
    z[H // 3:H // 3 + 9, W // 4:W // 4 + 9] = np.nan            # all-NaN windows for k <= 9
    z[:5, :5] = np.nan                                            # corner: NaN but for far taps
    z[-4:, -6:] = np.nan
    z[rng.random((H, W)) < 0.002] = np.inf
    z[rng.random((H, W)) < 0.002] = -np.inf
    return z


def _masks():
    ann = _circle(9) - _circle(9, 2)
    first_row_zero = np.ones((5, 7))
    first_row_zero[0] = 0
    odd_values = _circle(7)
    odd_values[1, 3] = 0.5                                        # neither 0.5 nor 2 is taken
    odd_values[3, 1] = 2.0
    return {"circle5": _circle(5), "annulus9": ann, "rect3x7": np.ones((3, 7)), "rect7x3": np.ones((7, 3)),
            "first_row_zero": first_row_zero, "values_0.5_2": odd_values, "circle25": _circle(25),
            "circle49": _circle(49)}


@pytest.mark.parametrize("name", list(_masks()))
def test_focal_stats_masks(lib, name):
    k = _masks()[name]
    for H, W in ((129, 260), (65, 132), (k.shape[0], 128), (2, 252)):
        _check_stats(lib, _raster(H, W, H + W + k.size), k, {}, "%s on %dx%d" % (name, H, W))
        _check_stats(lib, _signed_zero_raster(H, W, H * W), k, {}, "%s signed zeros on %dx%d" % (name, H, W))


@pytest.mark.parametrize("W", WIDTHS)
def test_focal_stats_widths_and_heights(lib, W):
    k = _circle(7)
    for H in _heights(7):
        _check_stats(lib, _signed_zero_raster(H, W, 3 * H + W), k, {}, "circle7 on %dx%d" % (H, W),
                     stats=("sum", "min", "max", "range", "mean"))


def test_focal_stats_pitched_and_offset_views(lib):
    k = _masks()["annulus9"]
    for W in (252, 2052):
        pad = (-(W * 4) % 128 + 16) // 4
        _check_stats(lib, _signed_zero_raster(67, W, W), k, {"pad_cols": pad}, "pitch +16 B, W %d" % W)
        _check_stats(lib, _signed_zero_raster(41, W, W + 1), k, {"rows_above": 3, "rows_below": 2},
                     "row-offset view, W %d" % W)


def test_min_max_keep_the_last_of_equal_zeros(lib):
    """Numba's nanmin / nanmax keep the LAST of equal cells in window order: [-0, +0] -> +0 and [+0, -0] -> -0
    for both min and max.  The tiled kernels must not order -0.0 below +0.0."""
    z = np.ones((64, 128), np.float32)
    z[10, 20], z[10, 21] = np.float32(-0.0), np.float32(0.0)
    z[30, 60], z[30, 61] = np.float32(0.0), np.float32(-0.0)
    k = np.ones((1, 3))
    for stat in ("min", "max", "range"):
        call = _stat_call(lib, k, stat)
        got = _launch(lib, lambda i, ip, out, op: call(i, ip, out, op, 64, 128), z, {}, K_STAT_TILED, stat)
        _bits_equal(got, o.focal_apply(z, k, stat), "%s tiled vs oracle" % stat)
    got = _launch(lib, lambda i, ip, out, op: _stat_call(lib, k, "min")(i, ip, out, op, 64, 128), z, {},
                  K_STAT_TILED, "min")
    assert not np.signbit(got[10, 21]), "window [-0, +0, 1]: min must be +0.0"
    assert np.signbit(got[30, 61]), "window [+0, -0, 1]: min must be -0.0"


@pytest.mark.parametrize("name", ["circle5", "annulus9", "first_row_zero", "circle25"])
def test_fused_focal_stats_bit_exact(lib, name):
    """The fused kernel (every statistic in one pass) against `apply` and the oracle: mean, sum, min, max and
    range bit for bit, var and std within the bound."""
    k = _masks()[name]
    kk = np.ascontiguousarray(k, dtype=np.float64)
    ids = np.array(list(STATS.values()), dtype=np.int32)
    for H, W in ((129, 260), (3, 132)):
        z = _signed_zero_raster(H, W, H + W + 1)
        t, ptr, pitch = _in_buffer(z)
        plane = (H * W * 4 + 15) // 16 * 16
        out = torch.full((len(ids) * plane // 4,), -1.0, dtype=torch.float32, device="cuda")
        lib.call("xrs_focal_stats_multi_f32", ptr, pitch, out.data_ptr(), W * 4, plane, H, W, kk.ctypes.data,
                 k.shape[0], k.shape[1], ids.ctypes.data, len(ids), _stream())
        torch.cuda.synchronize()
        assert lib.lib().xrs_debug_last_used_tma() == K_FUSED
        res = out.cpu().numpy()
        for i, (stat, sid) in enumerate(STATS.items()):
            got = res[i * plane // 4:i * plane // 4 + H * W].reshape(H, W)
            orc = o.focal_apply(z, k, stat, nthreads=o.max_threads())
            what = "fused %s %s %dx%d" % (stat, name, H, W)
            if stat in EXACT_STATS:
                _bits_equal(got, orc, what)
            else:
                _var_bound(got, orc, k, what)


def test_ragged_width_falls_back_per_plane(lib):
    """W % 4 != 0: no TMA, one bounds-checked launch per plane (the last one leaves code 8)."""
    H, W = 33, 130
    z = _signed_zero_raster(H, W, 5)
    k = _circle(5)
    kk = np.ascontiguousarray(k, dtype=np.float64)
    ids = np.array([0, 2, 3], dtype=np.int32)
    t, ptr, pitch = _in_buffer(z)
    plane = (H * W * 4 + 15) // 16 * 16
    out = torch.full((3 * plane // 4,), -1.0, dtype=torch.float32, device="cuda")
    lib.call("xrs_focal_stats_multi_f32", ptr, pitch, out.data_ptr(), W * 4, plane, H, W, kk.ctypes.data, 5, 5,
             ids.ctypes.data, 3, _stream())
    torch.cuda.synchronize()
    assert lib.lib().xrs_debug_last_used_tma() == K_STAT_DIRECT
    res = out.cpu().numpy()
    for i, stat in enumerate(("mean", "min", "max")):
        got = res[i * plane // 4:i * plane // 4 + H * W].reshape(H, W)
        _bits_equal(got, o.focal_apply(z, k, stat), "ragged %s" % stat)


# ------------------------------------------------------------------------------------------------ running box
def _box_rows(lib, H, W, kh, kw):
    """Rows where the launcher's row segments start (2 CTAs per SM, as launch_box_stream2 asks for), the
    raster's first and last kh rows, and the rows at both sides of a 4-row batch."""
    l = lib.lib()
    n = ctypes.c_int(0)
    lib.check(l.xrs_device_sm_count(0, ctypes.byref(n)))
    pad = (kw // 2 + 3) // 4 * 4
    n_tiles = (W + 7 * (128 - 2 * pad) - 1) // (7 * (128 - 2 * pad))
    seg = l.xrs_debug_pick_seg_rows(H, n_tiles, 2 * n.value, 12 * kh, kh - 1, 4, 4)
    rows = {0, 1, kh // 2, kh - 1, H - 1, H - 2, H - 1 - kh // 2, H - kh}
    for s in range(seg, H, seg):
        rows |= {s, s + 1, s - 1}
    return sorted(r for r in rows if 0 <= r < H), seg


@pytest.mark.parametrize("kw", range(5, 27, 2))
def test_running_box_magnitude_edges(lib, kw):
    """Uniform convolve_2d (w = 1/(kh kw) and -0.37) and focal.apply mean over all-ones windows, kh in {1, 3, kw},
    with cells from 2^24 M to FLT_MAX planted at segment starts, tile borders and raster edges: every window
    without a NaN / inf / planted cell stays within 2 ulp32 + 2^-36 |w| kh kw M of the tap-order oracle."""
    rng = np.random.default_rng(kw)
    W = 1028
    worst = 0.0
    for kh in sorted({1, 3, kw}):
        H = max(260, 26 * kh)                # row segments are at least 12 kh rows high
        fields = box_magnitude_fields(rng, H, W)
        rows, seg = _box_rows(lib, H, W, kh, kw)
        assert seg < H, "the raster should span more than one row segment"
        for field, z in fields.items():
            M = float(np.abs(z).max())
            for value in box_planted_values(M):
                data, planted = box_plant(z, value, rows, rng)
                for w in (1.0 / (kh * kw), -0.37):
                    k = np.full((kh, kw), w)
                    got = _launch(lib, lambda i, ip, out, op: _conv_call(lib, k)(i, ip, out, op, H, W), data, {},
                                  K_BOX, "box")
                    ref = o.convolve_2d_fma(data, k, nthreads=o.max_threads())
                    worst = max(worst, box_window_errors(got, ref, planted, kh, kw, w, M,
                                                         "convolve %dx%d %s %g w=%g" % (kh, kw, field, value, w)))
                ones = np.ones((kh, kw))
                got = _launch(lib, lambda i, ip, out, op: _stat_call(lib, ones, "mean")(i, ip, out, op, H, W),
                              data, {}, K_BOX, "box mean")
                ref = o.focal_apply(data, ones, "mean", nthreads=o.max_threads())
                worst = max(worst, box_window_errors(got, ref, planted, kh, kw, 1.0, M,
                                                     "mean %dx%d %s %g" % (kh, kw, field, value)))
    print("kw %d: worst clean-window error %.3g of the window scale" % (kw, worst))

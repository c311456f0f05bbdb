"""Where the 3x3 TMA kernel's bulk-store epilogue writes.

The TMA kernel stages each tile's output rows in shared memory and writes every row with one bulk copy of
min(tile width, W - x0) cells; rows outside a segment are skipped per row.  These tests call the C entry
points with a pitched output buffer prefilled with a sentinel and check two things: the cells inside the
H x W rectangle are bit-identical to what the cp.async kernel (register stores) computes from a
misaligned view of the same raster, and no byte outside the rectangle changed.  Runs on an H100 (`-m gpu`)."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

SENTINEL = 0x5A
# W % 4 == 0 throughout (the TMA path's condition); widths that are not a multiple of any tile width
# (1024 / 1536 / 2048 cells), widths below one tile, 1 / 2 / 3 / 5 rows, and heights cut into segments
SHAPES = [(1, 1028), (2, 1028), (3, 516), (5, 2052), (7, 8), (64, 132), (1000, 1028), (2053, 1036),
          (4099, 3000)]


@pytest.fixture(scope="module")
def lib():
    import xrspatial_b200
    assert torch.cuda.is_available(), "these tests need a CUDA device"
    return xrspatial_b200._lib


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _used_tma(lib):
    return lib.lib().xrs_debug_last_used_tma()


def _raster(H, W, seed):
    rng = np.random.default_rng(seed)
    z = rng.standard_normal((H, W)).cumsum(0).cumsum(1) * 3.0 + 500.0
    z[rng.random((H, W)) < 0.01] = np.nan
    return z.astype(np.float32)


def _aligned(z):
    """z on the device, contiguous (16-byte aligned rows when W % 4 == 0): the TMA path."""
    t = torch.from_numpy(np.ascontiguousarray(z)).cuda()
    return t, t.data_ptr(), t.stride(0) * t.element_size()


def _misaligned(z):
    """z on the device one element into a wider buffer: base and pitch not 16-byte aligned -> cp.async path."""
    H, W = z.shape
    big = torch.zeros((H, W + 1), dtype=torch.from_numpy(z[:0]).dtype, device="cuda")
    big[:, 1:] = torch.from_numpy(np.ascontiguousarray(z)).cuda()
    return big, big.data_ptr() + big.element_size(), big.stride(0) * big.element_size()


class Pitched(object):
    """An output rectangle of H x W cells inside a sentinel-filled buffer: one row above and below, 4 cells
    (16 or 32 bytes) left, 8 cells right, so the pitch stays a multiple of 16 bytes."""

    def __init__(self, H, W, itemsize):
        self.H, self.W, self.isz = H, W, itemsize
        self.wp = W + 12
        self.buf = torch.full(((H + 2) * self.wp * itemsize,), SENTINEL, dtype=torch.uint8, device="cuda")
        self.ptr = self.buf.data_ptr() + (self.wp + 4) * itemsize
        self.pitch = self.wp * itemsize

    def split(self):
        b = self.buf.cpu().numpy().reshape(self.H + 2, self.pitch)
        lo, hi = 4 * self.isz, (4 + self.W) * self.isz
        inside = b[1:1 + self.H, lo:hi].copy()
        b[1:1 + self.H, lo:hi] = SENTINEL
        return inside, b


def _check(lib, name, H, W, isz, tma_call, ref_call, kind=1):
    out = Pitched(H, W, isz)
    ref = torch.empty((H, W * isz), dtype=torch.uint8, device="cuda")
    tma_call(out.ptr, out.pitch)
    torch.cuda.synchronize()
    assert _used_tma(lib) == kind, "%s: TMA kernel was not selected" % name
    ref_call(ref.data_ptr(), W * isz)
    torch.cuda.synchronize()
    assert _used_tma(lib) == 0, "%s: the reference should take the cp.async kernel" % name
    inside, rest = out.split()
    np.testing.assert_array_equal(inside, ref.cpu().numpy(), err_msg="%s %dx%d: cells differ" % (name, H, W))
    bad = int((rest != SENTINEL).sum())
    assert bad == 0, "%s %dx%d: %d bytes outside the raster were written" % (name, H, W, bad)


def test_shapes_cut_short_segments(lib):
    """At least one of SHAPES leaves a short last segment for the segment heights the launcher picks."""
    l = lib.lib()
    n = ctypes.c_int(0)
    lib.check(l.xrs_device_sm_count(0, ctypes.byref(n)))
    short = False
    for H, W in SHAPES:
        # tile width, CTAs per SM and ROWS of the float32 operators, the float64-output focal means, the suite and
        # the int16 slope; make_tile_geom asks pick_seg_rows for ~2 waves
        for tile_w, ctas, rows in ((2048, 1, 4), (2048, 1, 2), (1536, 1, 8), (1024, 2, 4)):
            seg = l.xrs_debug_pick_seg_rows(H, (W + tile_w - 1) // tile_w, n.value * ctas, 32, 2, rows, 2)
            short |= H > seg and H % seg != 0
    assert short


@pytest.mark.parametrize("H,W", SHAPES)
def test_single_output_operators(lib, H, W):
    z = _raster(H, W, H * 7 + W)
    ta, pa, ia = _aligned(z)       # the tensors stay referenced while the kernels read them
    tm, pm, im = _misaligned(z)
    ex = np.array([np.nan], dtype=np.float64)
    ops = {
        "slope": lambda i, ip, o, op: lib.call("xrs_slope_f32", i, ip, o, op, H, W, 30.0, 30.0, _stream()),
        "slope aniso": lambda i, ip, o, op: lib.call("xrs_slope_f32", i, ip, o, op, H, W, 10.0, 25.5, _stream()),
        "aspect": lambda i, ip, o, op: lib.call("xrs_aspect_f32", i, ip, o, op, H, W, _stream()),
        "curvature": lambda i, ip, o, op: lib.call("xrs_curvature_f32", i, ip, o, op, H, W, 30.0, _stream()),
        "hillshade": lambda i, ip, o, op: lib.call("xrs_hillshade_f32", i, ip, o, op, H, W, 225.0, 25.0, _stream()),
        "focal.mean": lambda i, ip, o, op: lib.call("xrs_focal_mean_f32", i, ip, o, op, H, W,
                                                    ex.ctypes.data, 1, _stream()),
    }
    for name, fn in ops.items():
        _check(lib, name, H, W, 4, lambda o, op: fn(pa, ia, o, op), lambda o, op: fn(pm, im, o, op))
    # float32 in, float64 out
    fn = lambda i, ip, o, op: lib.call("xrs_focal_mean_f32_f64", i, ip, o, op, H, W,  # noqa: E731
                                       ex.ctypes.data, 1, _stream())
    _check(lib, "focal.mean f32->f64", H, W, 8, lambda o, op: fn(pa, ia, o, op), lambda o, op: fn(pm, im, o, op))
    # float64 in and out
    z64 = z.astype(np.float64)
    ta64, pa64, ia64 = _aligned(z64)
    tm64, pm64, im64 = _misaligned(z64)
    fn = lambda i, ip, o, op: lib.call("xrs_focal_mean_f64", i, ip, o, op, H, W,  # noqa: E731
                                       ex.ctypes.data, 1, _stream())
    _check(lib, "focal.mean f64", H, W, 8, lambda o, op: fn(pa64, ia64, o, op), lambda o, op: fn(pm64, im64, o, op))


@pytest.mark.parametrize("H,W", SHAPES)
def test_direct_ingest_int16(lib, H, W):
    """int16 rows read directly (pitch rounded up to 16 bytes) vs float32 hillshade of the cast raster."""
    z = np.round(_raster(H, W, H + 3 * W))
    z = np.nan_to_num(z, nan=-7.0).clip(-32768, 32767).astype(np.int16)
    wq = (W + 7) // 8 * 8
    zi = np.zeros((H, wq), dtype=np.int16)
    zi[:, :W] = z
    ti = torch.from_numpy(zi).cuda()
    tm, pm, im = _misaligned(z.astype(np.float32))
    par = np.array([225.0, 25.0])
    _check(lib, "hillshade int16", H, W, 4,
           lambda o, op: lib.call("xrs_surface_typed", 3, ti.data_ptr(), 4, wq * 2, o, op, H, W,
                                  par.ctypes.data, _stream()),
           lambda o, op: lib.call("xrs_hillshade_f32", pm, im, o, op, H, W, 225.0, 25.0, _stream()),
           kind=2)


@pytest.mark.parametrize("H,W", [(1, 1028), (5, 2052), (2053, 1036)])
def test_suite_with_null_outputs(lib, H, W):
    """The 4-output suite with aspect and curvature NULL: slope and hillshade land where they should and the
    NULL outputs cost no writes anywhere."""
    z = _raster(H, W, 99 + H)
    ta, pa, ia = _aligned(z)       # the tensors stay referenced while the kernels read them
    tm, pm, im = _misaligned(z)
    for which in ("slope", "hillshade"):
        def suite(i, ip, o, op, other):
            s, h = (o, other) if which == "slope" else (other, o)
            lib.call("xrs_surface_suite_f32", i, ip, s, None, None, h, op, H, W, 30.0, 30.0, 225.0, 25.0, _stream())
        side_t = Pitched(H, W, 4)
        side_r = Pitched(H, W, 4)
        _check(lib, "suite " + which, H, W, 4, lambda o, op: suite(pa, ia, o, op, side_t.ptr),
               lambda o, op: suite(pm, im, o, op, side_r.ptr))

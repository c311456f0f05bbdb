"""Where the 3x3 TMA kernel's bulk-store epilogue writes.

The TMA kernel stages each tile's output rows in shared memory and writes every row with one bulk copy of
min(tile width, W - x0) cells; rows outside a segment are skipped per row.  These tests call the C entry
points with a pitched output buffer prefilled with a sentinel and check two things: the cells inside the
H x W rectangle are bit-identical to what the cp.async kernel (register stores) computes from a
misaligned view of the same raster, and no byte outside the rectangle changed.  Runs on an H100 (`-m gpu`)."""
import ctypes

import numpy as np
import pytest

from helpers import K_INGEST, K_STRIP_CPASYNC, K_STRIP_TMA, Pitched, gpu_lib, in_buffer, last_kind, raster, stream

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

# W % 4 == 0 throughout (the TMA path's condition); widths that are not a multiple of any tile width
# (1024 / 1536 / 2048 cells), widths below one tile, 1 / 2 / 3 / 5 rows, and heights cut into segments
SHAPES = [(1, 1028), (2, 1028), (3, 516), (5, 2052), (7, 8), (64, 132), (1000, 1028), (2053, 1036),
          (4099, 3000)]


@pytest.fixture(scope="module")
def lib():
    return gpu_lib()


def _check(lib, name, H, W, isz, tma_call, ref_call, kind=K_STRIP_TMA):
    out = Pitched(H, W, isz)
    ref = torch.empty((H, W * isz), dtype=torch.uint8, device="cuda")
    tma_call(out.ptr, out.pitch)
    torch.cuda.synchronize()
    assert last_kind(lib) == kind, "%s: TMA kernel was not selected" % name
    ref_call(ref.data_ptr(), W * isz)
    torch.cuda.synchronize()
    assert last_kind(lib) == K_STRIP_CPASYNC, "%s: the reference should take the cp.async kernel" % name
    inside = out.inside("%s %dx%d" % (name, H, W))
    np.testing.assert_array_equal(inside, ref.cpu().numpy(), err_msg="%s %dx%d: cells differ" % (name, H, W))


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
    z = raster(H, W, H * 7 + W)
    ta, pa, ia = in_buffer(z)       # the tensors stay referenced while the kernels read them
    tm, pm, im = in_buffer(z, shift=1)
    ex = np.array([np.nan], dtype=np.float64)
    ops = {
        "slope": lambda i, ip, o, op: lib.call("xrs_slope_f32", i, ip, o, op, H, W, 30.0, 30.0, stream()),
        "slope aniso": lambda i, ip, o, op: lib.call("xrs_slope_f32", i, ip, o, op, H, W, 10.0, 25.5, stream()),
        "aspect": lambda i, ip, o, op: lib.call("xrs_aspect_f32", i, ip, o, op, H, W, stream()),
        "curvature": lambda i, ip, o, op: lib.call("xrs_curvature_f32", i, ip, o, op, H, W, 30.0, stream()),
        "hillshade": lambda i, ip, o, op: lib.call("xrs_hillshade_f32", i, ip, o, op, H, W, 225.0, 25.0, stream()),
        "focal.mean": lambda i, ip, o, op: lib.call("xrs_focal_mean_f32", i, ip, o, op, H, W,
                                                    ex.ctypes.data, 1, stream()),
    }
    for name, fn in ops.items():
        _check(lib, name, H, W, 4, lambda o, op: fn(pa, ia, o, op), lambda o, op: fn(pm, im, o, op))
    # float32 in, float64 out
    fn = lambda i, ip, o, op: lib.call("xrs_focal_mean_f32_f64", i, ip, o, op, H, W,  # noqa: E731
                                       ex.ctypes.data, 1, stream())
    _check(lib, "focal.mean f32->f64", H, W, 8, lambda o, op: fn(pa, ia, o, op), lambda o, op: fn(pm, im, o, op))
    # float64 in and out
    z64 = z.astype(np.float64)
    ta64, pa64, ia64 = in_buffer(z64)
    tm64, pm64, im64 = in_buffer(z64, shift=1)
    fn = lambda i, ip, o, op: lib.call("xrs_focal_mean_f64", i, ip, o, op, H, W,  # noqa: E731
                                       ex.ctypes.data, 1, stream())
    _check(lib, "focal.mean f64", H, W, 8, lambda o, op: fn(pa64, ia64, o, op), lambda o, op: fn(pm64, im64, o, op))


@pytest.mark.parametrize("H,W", SHAPES)
def test_direct_ingest_int16(lib, H, W):
    """int16 rows read directly (pitch rounded up to 16 bytes) vs float32 hillshade of the cast raster."""
    z = np.round(raster(H, W, H + 3 * W))
    z = np.nan_to_num(z, nan=-7.0).clip(-32768, 32767).astype(np.int16)
    wq = (W + 7) // 8 * 8
    zi = np.zeros((H, wq), dtype=np.int16)
    zi[:, :W] = z
    ti = torch.from_numpy(zi).cuda()
    tm, pm, im = in_buffer(z.astype(np.float32), shift=1)
    par = np.array([225.0, 25.0])
    _check(lib, "hillshade int16", H, W, 4,
           lambda o, op: lib.call("xrs_surface_typed", 3, ti.data_ptr(), 4, wq * 2, o, op, H, W,
                                  par.ctypes.data, stream()),
           lambda o, op: lib.call("xrs_hillshade_f32", pm, im, o, op, H, W, 225.0, 25.0, stream()),
           kind=K_INGEST)


@pytest.mark.parametrize("H,W", [(1, 1028), (5, 2052), (2053, 1036)])
def test_suite_with_null_outputs(lib, H, W):
    """The 4-output suite with aspect and curvature NULL: slope and hillshade land where they should and the
    NULL outputs cost no writes anywhere."""
    z = raster(H, W, 99 + H)
    ta, pa, ia = in_buffer(z)       # the tensors stay referenced while the kernels read them
    tm, pm, im = in_buffer(z, shift=1)
    for which in ("slope", "hillshade"):
        def suite(i, ip, o, op, other):
            s, h = (o, other) if which == "slope" else (other, o)
            lib.call("xrs_surface_suite_f32", i, ip, s, None, None, h, op, H, W, 30.0, 30.0, 225.0, 25.0, stream())
        side_t = Pitched(H, W, 4)
        side_r = Pitched(H, W, 4)
        _check(lib, "suite " + which, H, W, 4, lambda o, op: suite(pa, ia, o, op, side_t.ptr),
               lambda o, op: suite(pm, im, o, op, side_r.ptr))

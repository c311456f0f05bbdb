"""Where the 3x3 TMA kernel's input boxes start and end.

Each CTA tile reads its columns plus a 32-byte halo on each side (8 float32 cells, 16 two-byte cells, 4 float64
cells) in boxes of 208 cells; cells left of column 0 and right of W arrive as NaN (float maps) or are patched to
NaN from their coordinates (integer maps).  These tests compare the TMA kernels bit for bit with the cp.async
kernel, which fills its ring cell by cell with bounds checks, at widths around the halo, box and tile edges, on
pitched and row-offset inputs, and for every direct-ingest dtype.  Runs on an H100 (`-m gpu`)."""
import numpy as np
import pytest

from helpers import K_INGEST, K_STRIP_CPASYNC, K_STRIP_TMA, gpu_lib, in_buffer, last_kind, raster, stream

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

# below one box, one box +- a lane, around the 2048-cell tile of the 16-warp kernels, past two tiles
WIDTHS = [4, 252, 256, 260, 2044, 2052, 4100]
HEIGHTS = [1, 2, 3, 5, 67]


@pytest.fixture(scope="module")
def lib():
    return gpu_lib()


def _run(lib, fn, in_ptr, in_pitch, H, W, kind):
    out = torch.full((H, W), -1.0, dtype=torch.float32, device="cuda")
    fn(in_ptr, in_pitch, out.data_ptr(), W * 4)
    torch.cuda.synchronize()
    assert last_kind(lib) == kind
    return out.cpu().numpy().view(np.uint32)


def _ops(lib, H, W):
    ex = np.array([np.nan], dtype=np.float64)
    return {
        "slope": lambda i, ip, o, op: lib.call("xrs_slope_f32", i, ip, o, op, H, W, 30.0, 30.0, stream()),
        "hillshade": lambda i, ip, o, op: lib.call("xrs_hillshade_f32", i, ip, o, op, H, W, 225.0, 25.0, stream()),
        "focal.mean": lambda i, ip, o, op: lib.call("xrs_focal_mean_f32", i, ip, o, op, H, W,
                                                    ex.ctypes.data, 1, stream()),
        "suite": lambda i, ip, o, op: lib.call("xrs_surface_suite_f32", i, ip, None, None, None, o, op, H, W,
                                               30.0, 30.0, 225.0, 25.0, stream()),
    }


def _compare(lib, H, W, tma_view, seed):
    z = raster(H, W, seed)
    ta, pa, ia = in_buffer(z, **tma_view)    # the tensors stay referenced while the kernels read them
    tm, pm, im = in_buffer(z, shift=1)       # base not 16-byte aligned: the cp.async kernel
    for name, fn in _ops(lib, H, W).items():
        got = _run(lib, fn, pa, ia, H, W, K_STRIP_TMA)
        ref = _run(lib, fn, pm, im, H, W, K_STRIP_CPASYNC)
        np.testing.assert_array_equal(got, ref, err_msg="%s %dx%d %s: cells differ" % (name, H, W, tma_view))


@pytest.mark.parametrize("H", HEIGHTS)
@pytest.mark.parametrize("W", WIDTHS)
def test_widths_and_heights(lib, H, W):
    _compare(lib, H, W, {}, H * 131 + W)


@pytest.mark.parametrize("W", [252, 2052, 4100])
def test_pitch_not_multiple_of_128_bytes(lib, W):
    """Rows 16 bytes longer than a multiple of 128 B: box rows start 16 B into a sector on every other row."""
    pad = (-(W * 4) % 128 + 16) // 4
    _compare(lib, 37, W, {"pad_cols": pad}, W + 5)


@pytest.mark.parametrize("W", [256, 2044, 4100])
def test_row_offset_view(lib, W):
    """A stripe interior: the view starts rows into a larger raster, and the rows above and below it are other
    data, never read as the view's neighbours."""
    _compare(lib, 41, W, {"rows_above": 3, "rows_below": 2}, W + 11)


@pytest.mark.parametrize("dtype,code", [(np.int16, 4), (np.uint16, 5), (np.int32, 2), (np.float64, 1)])
@pytest.mark.parametrize("H,W", [(1, 4), (3, 252), (5, 260), (67, 2052), (9, 4100)])
def test_direct_ingest_edges(lib, dtype, code, H, W):
    """int16 / uint16 / int32 / float64 read directly at the left and right raster edges vs the float32 kernels
    on the cast raster (cp.async path); slope with rectangular cells and hillshade."""
    z = raster(H, W, 7 * H + W + code)
    if np.issubdtype(dtype, np.integer):
        lo = 0 if dtype == np.uint16 else -30000
        z = np.nan_to_num(np.round(z), nan=-7.0).clip(lo, 30000)
    zs = z.astype(dtype)
    wq = W + (-(W * zs.itemsize) % 16) // zs.itemsize   # pitch rounded up to 16 bytes
    buf = np.zeros((H, wq), dtype=dtype)
    buf[:, :W] = zs
    ts = torch.from_numpy(buf).cuda()
    tm, pm, im = in_buffer(zs.astype(np.float32), shift=1)
    cells = np.array([10.0, 25.5])
    sun = np.array([225.0, 25.0])
    cases = [
        ("slope", 0, cells, lambda o, op: lib.call("xrs_slope_f32", pm, im, o, op, H, W, 10.0, 25.5, stream())),
        ("hillshade", 3, sun, lambda o, op: lib.call("xrs_hillshade_f32", pm, im, o, op, H, W, 225.0, 25.0,
                                                     stream())),
    ]
    for name, op_code, par, ref_fn in cases:
        got = _run(lib, lambda i, ip, o, op: lib.call("xrs_surface_typed", op_code, i, code, ip, o, op, H, W,
                                                      par.ctypes.data, stream()),
                   ts.data_ptr(), wq * zs.itemsize, H, W, K_INGEST)
        ref = _run(lib, lambda i, ip, o, op: ref_fn(o, op), 0, 0, H, W, K_STRIP_CPASYNC)
        np.testing.assert_array_equal(got, ref, err_msg="%s %s %dx%d: cells differ" % (name, zs.dtype, H, W))

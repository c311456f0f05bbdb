"""The window sizes convolve_2d and the focal statistics accept: odd sides from 1 to 2047.  Everything else is
XRS_EINVAL with a message from each entry point, and from the host-raster entry point, before any CUDA
call, so these run without a GPU."""
import ctypes

import numpy as np
import pytest


@pytest.fixture(scope="module")
def xb():
    import xrspatial_b200
    return xrspatial_b200


BAD = [(2049, 3), (3, 2049), (2049, 2049), (4, 3), (3, 64), (2, 2)]


@pytest.mark.parametrize("kh,kw", BAD)
def test_entry_points_reject_the_window(xb, kh, kw):
    lib = xb._lib.lib()
    buf = (ctypes.c_float * 64)()
    src = ctypes.cast(buf, ctypes.c_void_p)
    dst = ctypes.c_void_p(ctypes.addressof(buf) + 128)
    k = (ctypes.c_double * (kh * kw))()
    kp = ctypes.cast(k, ctypes.c_void_p)
    ids = (ctypes.c_int * 2)(0, 3)
    words = b"too large" if max(kh, kw) > 2047 else b"odd"
    for rc in (lib.xrs_convolve2d_f32(src, 16, dst, 16, 2, 4, kp, kh, kw, None),
               lib.xrs_focal_stat_f32(src, 16, dst, 16, 2, 4, kp, kh, kw, 0, None),
               lib.xrs_focal_stats_multi_f32(src, 16, dst, 16, 32, 2, 4, kp, kh, kw, ids, 2, None)):
        assert rc == xb._lib.XRS_EINVAL
        assert words in lib.xrs_last_error_string()


def test_host_stencil_rejects_the_window(xb):
    _lib = xb._lib
    lib = _lib.lib()
    buf = (ctypes.c_float * 64)()
    ptr = ctypes.cast(buf, ctypes.c_void_p)
    dev = (ctypes.c_int * 1)(0)
    k = (ctypes.c_double * 9)()
    for op in (_lib.OPS["convolve"], _lib.OPS["focal_stat"]):
        for kh, kw in ((2049, 1), (1, 2049), (4, 1)):
            p = (ctypes.c_double * 3)(kh, kw, 0)
            assert lib.xrs_host_stencil(op, ptr, _lib.DTYPES["float32"], ptr, 4, 4, p, k, 9, dev, 1) \
                == _lib.XRS_EINVAL
            assert b"kernel" in lib.xrs_last_error_string()



def test_public_wrappers_raise_value_error(xb, monkeypatch):
    """Numpy rasters: the public wrappers reach xrs_host_stencil, which rejects the window before any CUDA call.
    The pinned result buffer is replaced by a plain one and the device list is given, so nothing here needs a
    GPU."""
    from xrspatial_b200 import _hostmem, focal
    from xrspatial_b200.convolution import convolution_2d, convolve_2d
    monkeypatch.setattr(_hostmem, "empty", np.empty)
    monkeypatch.setenv("XRS_B200_DEVICES", "0")
    z = np.zeros((6, 8), np.float32)
    agg = xb.DataArray(z, dims=("y", "x"), attrs={"res": (1, 1)})
    for k in (np.ones((2049, 1)), np.ones((1, 2049)), np.ones((2049, 2049))):
        for call in (lambda: convolve_2d(z, k), lambda: convolution_2d(agg, k), lambda: focal.apply(agg, k),
                     lambda: focal.apply(agg, k, func="max"),
                     lambda: focal.focal_stats(agg, k, stats_funcs=["mean", "max"])):
            with pytest.raises(ValueError, match="too large"):
                call()

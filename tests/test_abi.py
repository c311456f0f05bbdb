"""CPU-only: the C-ABI library loads and exports every symbol include/xrs_b200.h declares;
the product refuses to run without a CUDA device (no CPU fallback)."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "xrs_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(xrs_[a-z0-9_]+)\s*\(", src)))


def test_header_declares_the_hot_path():
    syms = header_symbols()
    for s in ("xrs_slope_f32", "xrs_aspect_f32", "xrs_curvature_f32", "xrs_hillshade_f32",
              "xrs_surface_suite_f32", "xrs_focal_mean_f32", "xrs_focal_mean_f64", "xrs_convolve2d_f32",
              "xrs_focal_stat_f32", "xrs_normalized_ratio_f32", "xrs_savi_f32", "xrs_evi_f32",
              "xrs_zonal_hash_run", "xrs_zonal_hash_second_pass", "xrs_host_stencil"):
        assert s in syms


def test_library_exports_every_declared_symbol_at_abi_version_3():
    import xrspatial_b200
    lib = xrspatial_b200._lib.lib()
    for s in header_symbols():
        assert hasattr(lib, s), "libxrs_b200.so does not export %s" % s
    assert lib.xrs_abi_version() == 3


def test_ctypes_prototypes_cover_the_header():
    import xrspatial_b200
    xrspatial_b200._lib.lib()
    declared = set(header_symbols()) - {"xrs_last_error_string"}
    assert declared <= set(xrspatial_b200._lib.EXPORTS), declared - set(xrspatial_b200._lib.EXPORTS)


def test_no_cpu_fallback_without_gpu():
    torch = pytest.importorskip("torch")
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    import xrspatial_b200 as xb
    agg = xb.DataArray(np.zeros((8, 8), np.float32), attrs={"res": (1, 1)})
    with pytest.raises(RuntimeError):
        xb.slope(agg)          # host path needs the device: fails loudly
    with pytest.raises(RuntimeError):
        xb.ndvi(agg, agg)


def test_argument_errors_do_not_need_a_gpu():
    import xrspatial_b200
    lib = xrspatial_b200._lib.lib()
    buf = (ctypes.c_float * 16)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    k = (ctypes.c_double * 4)(1, 1, 1, 1)
    # even kernel -> XRS_EINVAL before any CUDA call
    rc = lib.xrs_convolve2d_f32(p, 16, ctypes.c_void_p(ctypes.addressof(buf) + 32), 16, 2, 4,
                                ctypes.cast(k, ctypes.c_void_p), 2, 2, None)
    assert rc == -1
    assert b"odd" in lib.xrs_last_error_string()
    rc = lib.xrs_slope_f32(p, 8, p, 16, 2, 4, 1.0, 1.0, None)   # pitch < row bytes
    assert rc == -1
    with pytest.raises(ValueError):
        xrspatial_b200._lib.check(rc)


def test_host_stencil_rejects_bad_requests_before_any_cuda_call():
    """Every check of xrs_host_stencil runs before its first CUDA call: XRS_EINVAL (not XRS_ECUDA) and
    a message, also on a machine without a GPU."""
    import xrspatial_b200
    _lib = xrspatial_b200._lib
    lib = _lib.lib()
    F32, F64, I16 = _lib.DTYPES["float32"], _lib.DTYPES["float64"], _lib.DTYPES["int16"]
    OPS = _lib.OPS
    buf = (ctypes.c_double * (64 * 8))()
    ptr = ctypes.cast(buf, ctypes.c_void_p)
    p = (ctypes.c_double * 3)(3, 3, 0)
    k = (ctypes.c_double * 9)(*[1.0] * 9)

    def run(op, in_dtype, H=64, W=8, out=ptr, devices=(0,)):
        devs = (ctypes.c_int * len(devices))(*devices)
        return lib.xrs_host_stencil(op, ptr, in_dtype, out, H, W, p, k, 9, devs, len(devices))

    for args, kw, words in (((7, F32), {}, b"unknown op"),
                            ((8, F32), {}, b"unknown op"),
                            ((OPS["focal_mean"], I16), {}, b"focal mean"),
                            ((OPS["convolve"], F64), {}, b"convolve"),
                            ((OPS["slope"], I16), dict(W=6), b"W % 4"),
                            ((OPS["slope"], F32), dict(devices=(0, 0)), b"twice"),
                            ((OPS["slope"], F32), dict(out=None), b"NULL")):
        assert run(*args, **kw) == _lib.XRS_EINVAL, (args, kw)
        assert words in lib.xrs_last_error_string(), (args, kw, lib.xrs_last_error_string())
    assert run(OPS["slope"], F32, H=0) == _lib.XRS_OK

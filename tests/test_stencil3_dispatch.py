"""Dispatch of the 3x3 operators: every source cell type goes through one launcher, so int16 / uint16 / int32 /
float64 rasters (xrs_surface_typed) get the argument checks of the float32 entry points, and each (operator,
cell type) pair launches with its geometry.  The checks run on any machine; the geometry on an H100 (`-m gpu`)."""
import ctypes

import numpy as np
import pytest

from helpers import K_INGEST, K_STRIP_TMA, gpu_lib, last_kind, stream

torch = pytest.importorskip("torch")

TYPED = [("int16", 4, 2), ("uint16", 5, 2), ("int32", 2, 4), ("float64", 1, 8)]   # name, in_dtype, element size
H, W = 4, 8          # W % 4 == 0 and 16-byte rows for every cell type: a layout the TMA kernels take


@pytest.fixture(scope="module")
def clib():
    import xrspatial_b200
    return xrspatial_b200._lib


@pytest.fixture(scope="module")
def buf():
    """A 16-byte aligned 64 KB buffer, on the device when there is one, so that no case could touch host memory
    from a kernel even if its check were missing."""
    if torch.cuda.is_available():
        t = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    else:
        t = torch.zeros(1 << 16, dtype=torch.uint8)
    assert t.data_ptr() % 16 == 0
    return t


def _bad_calls(ptr, esz):
    """(what, in_pitch, out_pitch, in, out) of calls the launcher must refuse; pitches for `esz`-byte input cells,
    a valid in / out pair 4 KB apart."""
    other = ptr + 4096
    return [
        ("input pitch below the row", W * esz - esz, W * 4, ptr, other),
        ("input pitch not a multiple of the cell", W * esz + 1, W * 4, ptr, other),
        ("output pitch below the row", W * esz, W * 4 - 4, ptr, other),
        ("output pitch not a multiple of 4", W * esz, W * 4 + 2, ptr, other),
        ("in == out", W * esz, W * 4, ptr, ptr),
        ("out == NULL", W * esz, W * 4, ptr, None),
    ]


@pytest.mark.parametrize("name,code,esz", TYPED)
def test_typed_rasters_get_the_float32_argument_checks(clib, buf, name, code, esz):
    """xrs_surface_typed refuses what xrs_slope_f32 refuses, with the same status and message, before any CUDA
    call."""
    lib = clib.lib()
    p = (ctypes.c_double * 2)(10.0, 25.5)
    ptr = buf.data_ptr()
    typed = _bad_calls(ptr, esz)
    f32 = _bad_calls(ptr, 4)
    for (what, ip, op, i, o), (_, ip32, op32, i32, o32) in zip(typed, f32):
        for op_code in range(4):
            rc = lib.xrs_surface_typed(op_code, i, code, ip, o, op, H, W, p, None)
            msg = lib.xrs_last_error_string()
            rc32 = lib.xrs_slope_f32(i32, ip32, o32, op32, H, W, 10.0, 25.5, None)
            msg32 = lib.xrs_last_error_string()
            assert rc32 == clib.XRS_EINVAL, (what, msg32)
            assert (rc, msg) == (rc32, msg32), "%s, op %d, %s cells" % (what, op_code, name)


@pytest.mark.parametrize("name,code,esz", TYPED)
def test_typed_empty_rasters_do_nothing(clib, buf, name, code, esz):
    lib = clib.lib()
    p = (ctypes.c_double * 2)(10.0, 25.5)
    for h, w in ((0, W), (H, 0), (0, 0)):
        assert lib.xrs_surface_typed(0, buf.data_ptr(), code, W * esz, buf.data_ptr() + 4096, W * 4, h, w, p,
                                     None) == clib.XRS_OK


def test_typed_entry_point_leaves_float32_to_the_f32_entry_points(clib, buf):
    lib = clib.lib()
    p = (ctypes.c_double * 2)(10.0, 25.5)
    for op_code in range(4):
        rc = lib.xrs_surface_typed(op_code, buf.data_ptr(), clib.DTYPES["float32"], W * 4, buf.data_ptr() + 4096,
                                   W * 4, H, W, p, None)
        assert rc == clib.XRS_EUNSUPPORTED, op_code


# ----------------------------------------------------------------------------- geometry (H100)
# A raster with more tasks than resident CTAs for every geometry, so the grid is the resident CTA count:
# SMs x CTAs per SM.
GH, GW = 4096, 16384

# (kind, grid) recorded on an H100 80GB HBM3 (132 SMs, 700 W limit); a grid of 264 is two CTAs per SM
SMS = 132
GEOMETRY = {
    "slope f32 square cells": (K_STRIP_TMA, 132),
    "slope f32": (K_STRIP_TMA, 132),
    "aspect f32": (K_STRIP_TMA, 132),
    "curvature f32": (K_STRIP_TMA, 132),
    "hillshade f32": (K_STRIP_TMA, 132),
    "focal.mean f32": (K_STRIP_TMA, 132),
    "focal.mean f32 excludes": (K_STRIP_TMA, 132),
    "convolve 3x3": (K_STRIP_TMA, 132),
    "suite square cells": (K_STRIP_TMA, 132),
    "suite": (K_STRIP_TMA, 132),
    "focal.mean f64": (K_STRIP_TMA, 132),
    "focal.mean f32 -> f64": (K_STRIP_TMA, 132),
}
for _cells, _, _ in TYPED:
    GEOMETRY["slope %s" % _cells] = (K_INGEST, 264)
    for _op in ("aspect", "curvature", "hillshade"):
        GEOMETRY["%s %s" % (_op, _cells)] = (K_INGEST, 132)


def _launches(lib, src, src64, out, out64):
    """name -> a call that launches it on the raster"""
    c = lib.lib()
    s = stream()
    i, i64, o, o64 = src.data_ptr(), src64.data_ptr(), out.data_ptr(), out64.data_ptr()
    nan = (ctypes.c_double * 1)(float("nan"))
    ex = (ctypes.c_double * 2)(0.0, float("nan"))
    k3 = (ctypes.c_double * 9)(*[0.1 * (j + 1) for j in range(9)])
    pitch, pitch64 = GW * 4, GW * 8
    calls = {
        "slope f32 square cells": lambda: c.xrs_slope_f32(i, pitch, o, pitch, GH, GW, 30.0, 30.0, s),
        "slope f32": lambda: c.xrs_slope_f32(i, pitch, o, pitch, GH, GW, 10.0, 25.5, s),
        "aspect f32": lambda: c.xrs_aspect_f32(i, pitch, o, pitch, GH, GW, s),
        "curvature f32": lambda: c.xrs_curvature_f32(i, pitch, o, pitch, GH, GW, 30.0, s),
        "hillshade f32": lambda: c.xrs_hillshade_f32(i, pitch, o, pitch, GH, GW, 225.0, 25.0, s),
        "focal.mean f32": lambda: c.xrs_focal_mean_f32(i, pitch, o, pitch, GH, GW, nan, 1, s),
        "focal.mean f32 excludes": lambda: c.xrs_focal_mean_f32(i, pitch, o, pitch, GH, GW, ex, 2, s),
        "convolve 3x3": lambda: c.xrs_convolve2d_f32(i, pitch, o, pitch, GH, GW, k3, 3, 3, s),
        "suite square cells": lambda: c.xrs_surface_suite_f32(i, pitch, o, None, None, o64, pitch, GH, GW, 30.0,
                                                              30.0, 225.0, 25.0, s),
        "suite": lambda: c.xrs_surface_suite_f32(i, pitch, o, None, None, o64, pitch, GH, GW, 10.0, 25.5, 225.0,
                                                 25.0, s),
        "focal.mean f64": lambda: c.xrs_focal_mean_f64(i64, pitch64, o64, pitch64, GH, GW, nan, 1, s),
        "focal.mean f32 -> f64": lambda: c.xrs_focal_mean_f32_f64(i, pitch, o64, pitch64, GH, GW, nan, 1, s),
    }
    par = {"slope": (10.0, 25.5), "aspect": (0.0,), "curvature": (30.0,), "hillshade": (225.0, 25.0)}
    for cells, code, esz in TYPED:
        for op_code, op in enumerate(("slope", "aspect", "curvature", "hillshade")):
            p = (ctypes.c_double * 2)(*(par[op] + (0.0,))[:2])
            calls["%s %s" % (op, cells)] = (lambda op_code=op_code, code=code, esz=esz, p=p:
                                           c.xrs_surface_typed(op_code, i64, code, GW * esz, o, pitch, GH, GW, p, s))
    return calls


def observed_geometry(lib):
    """name -> (kind, grid) of every launch in GEOMETRY"""
    rng = np.random.default_rng(5)
    z = np.round(rng.standard_normal((GH, GW)).cumsum(1) * 3.0 + 500.0)
    src = torch.from_numpy(z.astype(np.float32)).cuda()
    src64 = torch.from_numpy(z).cuda()   # also read as int16 / uint16 / int32 cells: only the launch matters
    out = torch.empty((GH, GW), dtype=torch.float32, device="cuda")
    out64 = torch.empty((GH, GW), dtype=torch.float64, device="cuda")
    got = {}
    for name, call in _launches(lib, src, src64, out, out64).items():
        assert call() == 0, (name, lib.lib().xrs_last_error_string())
        got[name] = (last_kind(lib), lib.lib().xrs_debug_last_grid())
    torch.cuda.synchronize()
    return got


@pytest.mark.gpu
def test_every_operator_and_cell_type_launches_with_its_geometry():
    lib = gpu_lib()
    assert torch.cuda.get_device_properties(0).multi_processor_count == SMS, "the grids are those of a 132-SM H100"
    got = observed_geometry(lib)
    assert set(got) == set(GEOMETRY)
    bad = {k: (got[k], GEOMETRY[k]) for k in GEOMETRY if got[k] != GEOMETRY[k]}
    assert not bad, "(observed, expected): %s" % bad

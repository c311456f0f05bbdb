"""Raster arguments: the cell sets and argument checks every raster entry point shares (common.cuh), and the one
Python path from a raster to device cells (utils.device_cells): policies, broadcast rasters, uint64 widening and
scratch allocation failures."""
import ctypes
import importlib

import numpy as np
import pytest

import xrspatial_b200 as xb
from xrspatial_b200 import _lib, utils

H, W = 4, 8
RASTER, ZONAL, FLOAT = set(range(6)), set(range(11)), {0, 1}
CELL_SIZE = {0: 4, 1: 8, 2: 4, 3: 8, 4: 2, 5: 2, 6: 1, 7: 1, 8: 4, 9: 8, 10: 1, 11: 8}
_buf = (ctypes.c_double * 64)()
P = ctypes.cast(_buf, ctypes.c_void_p)   # never dereferenced: every call below fails an argument check first


def _need(query, *args):
    n = ctypes.c_int64()
    assert getattr(_lib.lib(), query)(*args, ctypes.byref(n)) == _lib.XRS_OK
    return n.value


def _i64():
    return ctypes.byref(ctypes.c_int64())


def _row(code, esz=None):
    return W * (CELL_SIZE[code] if esz is None else esz)


def _entry_points():
    """name: (cell set, output cell bytes of a code or None, call, the message of the check that follows the pitch
    checks).  call(code, in_pitch, out_pitch, last) passes the right pitches by default; with last=True the check
    after them fails (scratch one byte short, or an output pitch one cell short, or NULL values), so no call gets as
    far as the device."""
    L = _lib.lib()
    prox, vs, star = (_need(q, H, W, *a) for q, a in (("xrs_proximity_scratch_bytes", (0,)),
                                                        ("xrs_viewshed_scratch_bytes", ()),
                                                        ("xrs_a_star_scratch_bytes", ())))
    mom, sel = _need("xrs_classify_moments_scratch_bytes"), _need("xrs_classify_select_scratch_bytes")
    srt, reg = _need("xrs_classify_sort_scratch_bytes", H * W, 0), _need("xrs_zonal_regions_scratch_bytes", H, W)
    noise = _need("xrs_noise_scratch_bytes", H, W, 1)
    four, eight, own = (lambda c: 4), (lambda c: 8), (lambda c: CELL_SIZE[c])
    return {
        "xrs_proximity": (RASTER, four, lambda c, ip, op, last: L.xrs_proximity(
            P, c, ip, H, W, P, P, None, 0, 1.0, 0, 0, P, op, P, prox - last, 0, None), b"too small"),
        "xrs_viewshed": (RASTER, eight, lambda c, ip, op, last: L.xrs_viewshed(
            P, c, ip, H, W, 1, 1, 0.0, 0.0, 1.0, 1.0, P, op, P, vs - last, None), b"too small"),
        "xrs_a_star_search": (RASTER, eight, lambda c, ip, op, last: L.xrs_a_star_search(
            P, c, ip, H, W, P, 0, 8, 0, 0, 1, 1, P, op, P, star - last, None, None), b"too small"),
        "xrs_a_star_snap": (RASTER, None, lambda c, ip, op, last: L.xrs_a_star_snap(
            P, c, ip, H, W, P, 0, 0, 0, _i64(), _i64(), P, 256 - last, None), b"256 bytes"),
        "xrs_classify_cells": (RASTER, four, lambda c, ip, op, last: L.xrs_classify_cells(
            P, c, ip, H, W, 0, P, P, 1, P, op - 4 * last, None), b"output pitch"),
        "xrs_classify_moments": (RASTER, None, lambda c, ip, op, last: L.xrs_classify_moments(
            P, c, ip, H, W, 0.0, P, P, mom - last, None), b"too small"),
        "xrs_classify_select": (RASTER, None, lambda c, ip, op, last: L.xrs_classify_select(
            0, P, c, ip, H, W, 32, 0, None, 0, None, None, _i64(), P, P, sel - last, None), b"too small"),
        "xrs_classify_sort": (RASTER, None, lambda c, ip, op, last: L.xrs_classify_sort(
            P, c, ip, H, W, P, _i64(), P, srt - last, None), b"too small"),
        "xrs_zonal_regions": (ZONAL, own, lambda c, ip, op, last: L.xrs_zonal_regions(
            P, c, ip, H, W, 4, P, op, P, reg - last, None), b"too small"),
        "xrs_zonal_bounds": (ZONAL, None, lambda c, ip, op, last: L.xrs_zonal_bounds(
            P, c, ip, H, W, 0, None if last else P, None, 1, P, None), b"NULL values"),
        "xrs_noise": (FLOAT, own, lambda c, ip, op, last: L.xrs_noise(
            P, c, ip, H, W, P, P, P, 1, 1.0, P, op, P, P, noise - last, None), b"too small"),
    }


def _message():
    return _lib.lib().xrs_last_error_string()


def _call(entry, code, ip=None, op=None, last=True):
    out, call = entry[1], entry[2]
    return call(code, _row(code) if ip is None else ip, _row(code, out(code) if out else 8) if op is None else op,
                int(last))


@pytest.mark.parametrize("name", sorted(_entry_points()))
def test_every_cell_code_is_taken_or_refused_as_its_set_says(name):
    entry = _entry_points()[name]
    refused = b"float32 or float64" if name == "xrs_noise" else b"cell type"
    for code in range(12):
        assert _call(entry, code) == _lib.XRS_EINVAL, (name, code)
        assert (entry[3] if code in entry[0] else refused) in _message(), (name, code, _message())


@pytest.mark.parametrize("name", sorted(_entry_points()))
def test_pitches_one_cell_short_or_off_the_cell_size_are_refused(name):
    entry = _entry_points()[name]
    cells, out = entry[:2]
    for code in sorted(cells):
        esz = CELL_SIZE[code]
        for ip in [_row(code) - esz] + ([_row(code) + 1] if esz > 1 else []):
            assert _call(entry, code, ip=ip, last=False) == _lib.XRS_EINVAL
            assert b"input pitch" in _message(), (name, code, ip, _message())
        if out is None:
            continue
        osz = out(code)
        for op in [_row(code, osz) - osz] + ([_row(code, osz) + 1] if osz > 1 else []):
            assert _call(entry, code, op=op, last=False) == _lib.XRS_EINVAL
            assert b"output pitch" in _message(), (name, code, op, _message())


@pytest.mark.parametrize("name", sorted(n for n, e in _entry_points().items() if e[3] in (b"too small", b"256 bytes")))
def test_scratch_one_byte_short_is_too_small(name):
    entry = _entry_points()[name]
    for code in sorted(entry[0]):
        assert _call(entry, code) == _lib.XRS_EINVAL
        assert entry[3] in _message() and (name == "xrs_a_star_snap" or b"_scratch_bytes)" in _message())


# ----------------------------------------------------------------------------- the Python cell policies
@pytest.mark.parametrize("dtype, widen, as_is, floats", [
    ("float32", "float32", "float32", "float32"), ("float64", "float64", "float64", "float64"),
    ("int16", "int16", "int16", None), ("uint16", "uint16", "uint16", None), ("int32", "int32", "int32", None),
    ("int64", "int64", "int64", None), ("bool", "int16", "bool", None), ("int8", "int16", "int8", None),
    ("uint8", "int16", "uint8", None), ("uint32", "int64", "uint32", None), ("uint64", "int64", "uint64", None),
    ("float16", "float32", None, None), ("complex64", None, None, None)])
def test_cell_policies_on_numpy_rasters(dtype, widen, as_is, floats):
    z = (np.arange(12).reshape(3, 4) % 3).astype(dtype)
    for policy, want, error in (("widen", widen, TypeError), ("as-is", as_is, NotImplementedError),
                                ("float", floats, TypeError)):
        if want is None:
            with pytest.raises(error):
                utils.raster_cells(z, "f", policy)
            continue
        cells, code = utils.raster_cells(z, "f", policy)
        assert cells.dtype == np.dtype(want) and code == _lib.ZONAL_CELLS[want]
        assert np.array_equal(cells, z)


def test_raster_checks_before_any_device_work():
    with pytest.raises(ValueError, match="above 2\\*\\*63"):
        utils.raster_cells(np.array([[1, 2 ** 63]], np.uint64), "proximity", "widen")
    with pytest.raises(ValueError, match="2-D"):
        utils.raster_cells(np.zeros(4, np.float32), "f", "widen")
    with pytest.raises(TypeError, match="Unsupported raster array type"):
        utils.raster_cells([[1.0]], "f", "widen")
    with pytest.raises(NotImplementedError, match="Dask"):
        utils.raster_cells(type("A", (), {"__module__": "dask.array.core"})(), "f", "widen")


# ----------------------------------------------------------------------------- on the device
def _da(data):
    h, w = data.shape
    return xb.DataArray(data, dims=("y", "x"), coords={"y": np.arange(h, dtype=np.float64),
                                                       "x": np.arange(w, dtype=np.float64)}, attrs={"res": (1.0, 1.0)})


def _same(a, b):
    import torch
    torch.testing.assert_close(a, b, rtol=0, atol=0, equal_nan=True)


@pytest.mark.gpu
def test_broadcast_rasters_give_the_contiguous_result():
    import torch
    row = torch.tensor([0, 0, 3, 0, 5, 5, 0, 2, 0, 1, 0, 0], dtype=torch.float32, device="cuda")
    for h in (1, 7):
        b = row.expand(h, row.numel())
        assert b.stride(0) == 0 or h == 1
        c = b.contiguous()
        runs = [lambda d: xb.proximity(_da(d)).data, lambda d: xb.viewshed(_da(d), x=3.0, y=0.0).data,
                lambda d: xb.a_star_search(_da(d), (0.0, 0.0), (h - 1.0, 11.0)).data,
                lambda d: xb.quantile(_da(d), k=3).data, lambda d: xb.regions(_da(d)).data]
        for run in runs:
            _same(run(b), run(c))


@pytest.mark.gpu
def test_torch_uint64_rasters_follow_the_numpy_rule():
    import torch
    z = np.array([[0, 3, 0, 9], [2 ** 40, 0, 0, 2 ** 63 - 1]], np.uint64)
    got = xb.proximity(_da(torch.from_numpy(z).cuda()), target_values=[3, 2 ** 40]).data
    want = xb.proximity(_da(torch.from_numpy(z.astype(np.int64)).cuda()), target_values=[3, 2 ** 40]).data
    _same(got, want)
    _same(got.cpu(), torch.from_numpy(xb.proximity(_da(z), target_values=[3, 2 ** 40]).data))
    z[0, 0] = 2 ** 63
    with pytest.raises(ValueError, match="above 2\\*\\*63"):
        xb.proximity(_da(torch.from_numpy(z).cuda()))


@pytest.mark.gpu
def test_failed_scratch_allocations_raise_memory_error(monkeypatch):
    import torch
    classify, perlin = (importlib.import_module("xrspatial_b200." + m) for m in ("classify", "perlin"))
    z = torch.arange(48, dtype=torch.float32, device="cuda").reshape(6, 8) % 5
    real = torch.empty

    def empty(*shape, dtype=None, **kw):   # every scratch buffer is uint8; nothing else on these paths is
        if dtype is torch.uint8:
            raise torch.OutOfMemoryError("CUDA out of memory (test)")
        return real(*shape, dtype=dtype, **kw)

    monkeypatch.setattr(torch, "empty", empty)
    calls = [lambda: xb.proximity(_da(z)), lambda: xb.viewshed(_da(z), x=1.0, y=1.0),
             lambda: xb.a_star_search(_da(z + 1), (0.0, 0.0), (5.0, 7.0)), lambda: xb.regions(_da(z)),
             lambda: xb.quantile(_da(z), k=3), lambda: classify.sample_indices(1000, 10, z.device),
             lambda: classify.jenks_matrices(real(16, dtype=torch.float32, device="cuda"), 3),
             lambda: perlin.perm_tables([1], z.device)]
    for call in calls:
        with pytest.raises(MemoryError, match="bytes of device scratch"):
            call()

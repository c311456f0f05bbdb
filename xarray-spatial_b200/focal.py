"""xrspatial.focal on the CUDA backend (reference: focal.py): mean, apply, focal_stats.

`apply` accepts the built-in reducers only (`_calc_mean`, `_calc_sum`, ... or their names): an
arbitrary Python/Numba callable cannot cross the C ABI (SURVEY.md section 2 row 7).
`hotspots` (SURVEY.md section 8f rank 1) = convolve_2d + global mean/std + an int8 classification.
"""
import ctypes
from collections import OrderedDict

import numpy as np
import pandas as pd

from . import _lib
from ._xr import DataArray, concat
from .convolution import custom_kernel
from .dataset_support import supports_dataset
from .utils import (ArrayTypeFunctionMapping, _dbl_array, as_device_tensor, call_on, device_2d, is_device_array,
                    like_container, pitch, ptr, run_stencil_device, run_stencil_host)


class _Reducer(object):
    """Named window reducer; stands in for the reference's @ngjit `_calc_*` functions."""

    def __init__(self, stat):
        self.stat = stat
        self.__name__ = "_calc_" + stat

    def __repr__(self):
        return "<focal reducer %s>" % self.stat


_calc_mean = _Reducer("mean")
_calc_sum = _Reducer("sum")
_calc_min = _Reducer("min")
_calc_max = _Reducer("max")
_calc_std = _Reducer("std")
_calc_range = _Reducer("range")
_calc_var = _Reducer("var")
_REDUCERS = {r.stat: r for r in (_calc_mean, _calc_sum, _calc_min, _calc_max, _calc_std,
                                 _calc_range, _calc_var)}


def _stat_of(func):
    if isinstance(func, _Reducer):
        return func.stat
    if isinstance(func, str) and func in _REDUCERS:
        return func
    name = getattr(func, "__name__", "")
    if name.startswith("_calc_") and name[6:] in _REDUCERS:
        return name[6:]
    raise NotImplementedError(
        "focal.apply on the CUDA backend supports the built-in reducers only "
        "(mean, sum, min, max, std, range, var); got %r" % (func,))


# ----------------------------------------------------------------------------- mean
def _mean_numpy(data, excludes):
    """One pass on a host raster, float64 result (replaces focal.py:44 `_mean_numpy` after the
    `astype(float)` of focal.py:257; a float32 raster is widened inside the kernel)."""
    return run_stencil_host("focal_mean", data, aux=tuple(excludes))


def _mean_cupy(data, excludes):
    """One pass on a device raster (replaces focal.py:135 `_mean_cupy`): float32 like the
    reference's GPU path, float64 if the input is float64."""
    import torch
    ex = _dbl_array(tuple(excludes))
    if as_device_tensor(data).dtype == torch.float64:
        return run_stencil_device(data, "xrs_focal_mean_f64", ex, len(excludes), cells=("float64",), out="float64")
    return run_stencil_device(data, "xrs_focal_mean_f32", ex, len(excludes))


def _mean(data, excludes):
    mapper = ArrayTypeFunctionMapping(numpy_func=_mean_numpy, cupy_func=_mean_cupy)
    return mapper(DataArray(data))(data, excludes)


@supports_dataset
def mean(agg, passes=1, excludes=[np.nan], name='mean'):
    """3x3 NaN-skipping mean filter applied `passes` times; cells equal to an `excludes` value
    are passed through (focal.py:162-265).  numpy-backed input -> float64 like the reference's
    CPU path; device input -> float32 (float64 if the input is float64) like its GPU path."""
    data = agg.data
    excludes = tuple(excludes)
    if len(excludes) > 8:
        raise ValueError("at most 8 exclude values are supported")
    if isinstance(data, np.ndarray):
        if passes <= 1:
            out = data.astype(float) if passes < 1 else _mean_numpy(data, excludes)
        else:
            # keep intermediate passes on the device: one upload, `passes` kernels, one download
            import torch
            cur = device_2d(data, torch.float64)
            for _ in range(passes):
                cur = _mean_cupy(cur, excludes)
            out = cur.cpu().numpy()
    elif is_device_array(data):
        import torch
        cur = as_device_tensor(data)
        if cur.dtype not in (torch.float32, torch.float64):
            cur = cur.to(torch.float32)
        for _ in range(passes):
            cur = _mean_cupy(cur, excludes)
        out = like_container(cur, data)
    else:
        out = _mean(data, excludes)  # raises for unsupported kinds
    return DataArray(out, name=name, dims=agg.dims, coords=agg.coords, attrs=agg.attrs)


# ----------------------------------------------------------------------------- apply / stats
def _apply_numpy(data, kernel, func):
    """replaces focal.py:305 `_apply_numpy` (host raster)."""
    k = np.ascontiguousarray(kernel, dtype=np.float64)
    return run_stencil_host("focal_stat", data, (k.shape[0], k.shape[1], _lib.STATS[_stat_of(func)]),
                            aux=k.ravel())


def _apply_cupy(data, kernel, func):
    """device raster -> xrs_focal_stat_f32 with the CPU (NaN-skipping) semantics."""
    k = np.ascontiguousarray(kernel, dtype=np.float64)
    return run_stencil_device(data, "xrs_focal_stat_f32", k.ctypes.data_as(ctypes.c_void_p), k.shape[0], k.shape[1],
                              _lib.STATS[_stat_of(func)])


def apply(raster, kernel, func=_calc_mean, name='focal_apply'):
    """Reducer over the cells where `kernel == 1`, NaN and out-of-raster cells skipped
    (focal.py:343-473)."""
    if not isinstance(raster, DataArray):
        raise TypeError("`raster` must be instance of DataArray")
    if raster.ndim != 2:
        raise ValueError("`raster` must be 2D")
    kernel = custom_kernel(kernel)
    mapper = ArrayTypeFunctionMapping(numpy_func=_apply_numpy, cupy_func=_apply_cupy)
    out = mapper(raster)(raster.data, kernel, func)
    return DataArray(out, name=name, coords=raster.coords, dims=raster.dims, attrs=raster.attrs)


def _focal_stats_cupy(data, kernel, stats_funcs):
    """device raster -> (stats, y, x) stack from ONE pass (xrs_focal_stats_multi_f32); replaces
    focal.py:757 `_focal_stats_cupy`, with the CPU (NaN-skipping, kernel == 1) semantics."""
    import torch
    t = device_2d(data, torch.float32)
    H, W = t.shape
    k = np.ascontiguousarray(kernel, dtype=np.float64)
    ids = (ctypes.c_int * len(stats_funcs))(*[_lib.STATS[s] for s in stats_funcs])
    plane = (H * W + 3) // 4 * 4          # planes start on 16-byte boundaries
    out = torch.empty(len(stats_funcs) * plane, dtype=torch.float32, device=t.device)
    out = out.as_strided((len(stats_funcs), H, W), (plane, W, 1))
    if H and W:   # the row and the plane pitch of the stack
        call_on(t, "xrs_focal_stats_multi_f32", ptr(t), pitch(t), ptr(out), pitch(out[0]), pitch(out), H, W,
                k.ctypes.data_as(ctypes.c_void_p), k.shape[0], k.shape[1], ids, len(stats_funcs))
    return like_container(out, data)


def focal_stats(agg, kernel, stats_funcs=['mean', 'max', 'min', 'range', 'std', 'var', 'sum']):
    """Stack of focal statistics along a new 'stats' dimension (focal.py:800-878)."""
    if not isinstance(agg, DataArray):
        raise TypeError("`agg` must be instance of DataArray")
    if agg.ndim != 2:
        raise ValueError("`agg` must be 2D")
    kernel = custom_kernel(kernel)
    for stats in stats_funcs:
        if stats not in _REDUCERS:
            raise ValueError("unknown focal statistic %r" % (stats,))
    stats_funcs = list(stats_funcs)
    index = pd.Index(stats_funcs, name='stats', dtype=object)
    if stats_funcs and is_device_array(agg.data) and len(set(stats_funcs)) == len(stats_funcs):
        # one call writing straight into the stacked result (the C entry point rejects a repeated statistic)
        data = _focal_stats_cupy(agg.data, kernel, stats_funcs)
        coords = OrderedDict()
        coords['stats'] = np.asarray(stats_funcs, dtype=object)
        coords.update(agg.coords)
        return DataArray(data, coords=coords, dims=('stats',) + tuple(agg.dims), attrs=agg.attrs,
                         name='focal_apply')
    stats_aggs = [apply(agg, kernel, func=_REDUCERS[stats]) for stats in stats_funcs]
    return concat(stats_aggs, index)


# ----------------------------------------------------------------------------- hotspots
def _hotspots_device(data, kernel):
    """convolve with kernel / kernel.sum(), z-score against the raster's global NaN-skipping
    mean / std, classify (replaces focal.py:918-937 `_hotspots_numpy` / :1025 `_hotspots_cupy`)."""
    import torch
    from .convolution import _convolve_2d_cupy
    t = device_2d(data, torch.float32)
    k = np.asarray(kernel, dtype=np.float64)
    mean_array = as_device_tensor(_convolve_2d_cupy(t, k / k.sum()))
    part = torch.empty(3, dtype=torch.float64, device=t.device)
    tc = t.contiguous()
    flat = tc.reshape(-1)
    step = max(1, flat.numel() // 65536)
    sample = flat[::step]
    sample = sample[~torch.isnan(sample)]
    pivot = float(sample.double().mean().item()) if sample.numel() else 0.0
    call_on(tc, "xrs_global_stats_f32", ptr(tc), tc.numel(), pivot, ptr(part))
    cnt, s1, s2 = [float(x) for x in part.cpu().numpy()]
    if cnt == 0:
        gmean = gstd = float("nan")
    else:
        gmean = pivot + s1 / cnt
        gstd = float(np.sqrt(max(s2 / cnt - (s1 / cnt) ** 2, 0.0)))
    if gstd == 0:
        raise ZeroDivisionError("Standard deviation of the input raster values is 0.")
    out = torch.empty(tuple(t.shape), dtype=torch.int8, device=t.device)
    m = mean_array.contiguous()
    call_on(m, "xrs_hotspots_classify_f32", ptr(m), m.numel(), float(np.float32(gmean)), float(np.float32(gstd)),
            ptr(out))
    return out


def hotspots(raster, kernel):
    """Getis-Ord Gi* hot / cold spots: int8 confidence levels in {0, +-90, +-95, +-99}
    (focal.py:1050-1125)."""
    import copy
    if not isinstance(raster, DataArray):
        raise TypeError("`raster` must be instance of DataArray")
    if raster.ndim != 2:
        raise ValueError("`raster` must be 2D")
    kind = getattr(raster.data.dtype, "kind", None)
    if kind is not None and kind not in "iuf":
        raise ValueError("data type must be integer or float")
    if isinstance(raster.data, np.ndarray):
        out = _hotspots_device(raster.data, kernel).cpu().numpy()
    elif is_device_array(raster.data):
        out = like_container(_hotspots_device(raster.data, kernel), raster.data)
    else:
        raise TypeError("Unsupported Array Type: {}".format(type(raster.data)))
    attrs = copy.deepcopy(raster.attrs)
    attrs['unit'] = '%'
    return DataArray(out, coords=raster.coords, dims=raster.dims, attrs=attrs)

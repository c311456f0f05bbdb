"""proximity, allocation and direction (proximity.py:24-1072 of the reference) on the GPU.

Each cell gets the target nearest to it under the metric, exactly: among equidistant targets, the first in
row-major order.  The reference's GDAL-style sweep (proximity.py:261-398) passes a target to a cell only through
its neighbours and can miss the nearest one; where it finds it, the outputs are equal (DESIGN.md section 4.7).
The distance, allocation and direction values follow the reference's formulas and float32 roundings.
"""
import ctypes

import numpy as np

from . import _lib
from ._xr import DataArray
from .dataset_support import supports_dataset
from .utils import device_2d, is_dask_array, is_device_array, like_container, stream_ptr

EUCLIDEAN = 0
GREAT_CIRCLE = 1
MANHATTAN = 2

PROXIMITY = 0
ALLOCATION = 1
DIRECTION = 2

DISTANCE_METRICS = {"EUCLIDEAN": EUCLIDEAN, "GREAT_CIRCLE": GREAT_CIRCLE, "MANHATTAN": MANHATTAN}

# numpy cell types the kernels read as they are, and the type each other one is widened to without changing a value
_DTYPE_CODES = {np.dtype(k): v for k, v in _lib.DTYPES.items()}
_WIDEN = {np.dtype(np.bool_): np.int16, np.dtype(np.int8): np.int16, np.dtype(np.uint8): np.int16,
          np.dtype(np.uint32): np.int64, np.dtype(np.uint64): np.int64, np.dtype(np.float16): np.float32}


def euclidean_distance(x1: float, x2: float, y1: float, y2: float) -> float:
    """Straight-line distance between (x1, y1) and (x2, y2)."""
    x = x1 - x2
    y = y1 - y2
    return np.sqrt(x * x + y * y)


def manhattan_distance(x1: float, x2: float, y1: float, y2: float) -> float:
    """Sum of the distances along x and y between (x1, y1) and (x2, y2)."""
    x = x1 - x2
    y = y1 - y2
    return abs(x) + abs(y)


def _check_lon_lat(x1, x2, y1, y2):
    if x1 > 180 or x1 < -180:
        raise ValueError("Invalid x-coordinate of the first point.Must be in the range [-180, 180]")
    if x2 > 180 or x2 < -180:
        raise ValueError("Invalid x-coordinate of the second point.Must be in the range [-180, 180]")
    if y1 > 90 or y1 < -90:
        raise ValueError("Invalid y-coordinate of the first point.Must be in the range [-90, 90]")
    if y2 > 90 or y2 < -90:
        raise ValueError("Invalid y-coordinate of the second point.Must be in the range [-90, 90]")


def great_circle_distance(x1: float, x2: float, y1: float, y2: float, radius: float = 6378137) -> float:
    """Haversine distance between the (longitude, latitude) points (x1, y1) and (x2, y2) on a sphere of `radius`."""
    _check_lon_lat(x1, x2, y1, y2)
    lat1, lon1, lat2, lon2 = np.radians(y1), np.radians(x1), np.radians(y2), np.radians(x2)
    dlon = lon2 - lon1
    dlat = lat2 - lat1
    a = np.sin(dlat / 2.0) ** 2 + np.cos(lat1) * np.cos(lat2) * np.sin(dlon / 2.0) ** 2
    return radius * 2 * np.arcsin(np.sqrt(a))


def _monotone(v, name):
    d = np.diff(v)
    if v.ndim != 1 or not (np.all(d > 0) or np.all(d < 0)) or not np.all(np.isfinite(v)):
        raise NotImplementedError(
            "proximity needs the 1-D coordinate %r to be finite and strictly ascending or descending" % name)


def _coord(raster, name):
    c = raster[name]
    return np.ascontiguousarray(getattr(c, "data", c), dtype=np.float64)


def _cells(data):
    """The raster as a 2-D CUDA tensor of one of the library's cell types, and that type's code."""
    import torch
    if isinstance(data, np.ndarray):
        widen = _WIDEN.get(data.dtype)
        if data.dtype == np.uint64 and data.size and data.max() > np.iinfo(np.int64).max:
            raise ValueError("uint64 cells above 2**63 - 1 are not supported")
        if widen is not None:
            data = data.astype(widen)
        if data.dtype not in _DTYPE_CODES:
            raise TypeError("unsupported cell type %s" % data.dtype)
        t = device_2d(data)
    else:
        t = device_2d(data)
        widen = {torch.bool: torch.int16, torch.int8: torch.int16, torch.uint8: torch.int16,
                 torch.uint32: torch.int64, torch.float16: torch.float32, torch.bfloat16: torch.float32}
        if t.dtype in widen:
            t = t.to(widen[t.dtype])
    code = _lib.DTYPES.get(str(t.dtype).replace("torch.", ""))
    if code is None:
        raise TypeError("unsupported cell type %s" % t.dtype)
    return t, code


def _process(raster, x, y, target_values, max_distance, distance_metric, process_mode, band_rows=0):
    """The transform behind proximity / allocation / direction (proximity.py:401-647): float32 raster of the
    distance, the nearest target's value or the direction to it.  `band_rows` (0: the library's choice) only
    sets how the column pass is split; the result does not depend on it."""
    import torch
    if tuple(raster.dims) != (y, x):
        raise ValueError("raster.coords should be named as coordinates:({0}, {1})".format(y, x))
    metric = DISTANCE_METRICS.get(distance_metric, EUCLIDEAN)
    if max_distance is None:
        max_distance = np.inf
    data = raster.data
    if is_dask_array(data):
        raise NotImplementedError("proximity: Dask arrays are not supported by the GPU backend")
    if not (isinstance(data, np.ndarray) or is_device_array(data)):
        raise TypeError("Unsupported Array Type: {}".format(type(data)))
    xs, ys = _coord(raster, x), _coord(raster, y)
    _monotone(xs, x)
    _monotone(ys, y)
    if metric == GREAT_CIRCLE and xs.size and ys.size:
        _check_lon_lat(xs.min(), xs.max(), ys.min(), ys.max())
    t, code = _cells(data)
    H, W = t.shape
    if (len(xs), len(ys)) != (W, H):
        raise ValueError("coordinate lengths (%d, %d) do not match the raster's shape %s" % (len(ys), len(xs), (H, W)))
    out = torch.empty((H, W), dtype=torch.float32, device=t.device)
    if H and W:
        tv = np.asarray(target_values)
        targets = None
        if tv.size:
            vals = np.unique(tv.astype(np.float64).ravel())   # NumPy compares the cells with them in float64
            vals = vals[~np.isnan(vals)]
            # never a NULL list (the default rule), also when no value can match
            targets = torch.as_tensor(np.append(vals, 0.0), device=t.device)[:vals.size]
        need = ctypes.c_int64()
        _lib.call("xrs_proximity_scratch_bytes", H, W, int(band_rows), ctypes.byref(need))
        scratch = torch.empty(need.value, dtype=torch.uint8, device=t.device)
        xt = torch.as_tensor(xs, device=t.device)
        yt = torch.as_tensor(ys, device=t.device)
        with torch.cuda.device(t.device):
            _lib.call("xrs_proximity", ctypes.c_void_p(t.data_ptr()), code, t.stride(0) * t.element_size(), H, W,
                      ctypes.c_void_p(xt.data_ptr()), ctypes.c_void_p(yt.data_ptr()),
                      None if targets is None else ctypes.c_void_p(targets.untyped_storage().data_ptr()),
                      0 if targets is None else vals.size, float(max_distance), metric, int(process_mode),
                      ctypes.c_void_p(out.data_ptr()), out.stride(0) * 4, ctypes.c_void_p(scratch.data_ptr()),
                      need.value, int(band_rows), stream_ptr(t))
    if isinstance(data, np.ndarray):
        return out.cpu().numpy()
    return like_container(out, data)


def _wrap(result, raster):
    return DataArray(result, coords=raster.coords, dims=raster.dims, attrs=raster.attrs)


@supports_dataset
def proximity(raster, x="x", y="y", target_values=[], max_distance=np.inf, distance_metric="EUCLIDEAN"):
    """Distance from every cell to the nearest target cell (proximity.py:652-790).  Targets are the cells equal
    to one of `target_values`, or every nonzero finite cell when it is empty; distances beyond `max_distance`
    are NaN.  float32, with the input's coords, dims and attrs."""
    return _wrap(_process(raster, x, y, target_values, max_distance, distance_metric, PROXIMITY), raster)


@supports_dataset
def allocation(raster, x="x", y="y", target_values=[], max_distance=np.inf, distance_metric="EUCLIDEAN"):
    """Value of the nearest target cell for every cell (proximity.py:793-928), NaN beyond `max_distance`."""
    return _wrap(_process(raster, x, y, target_values, max_distance, distance_metric, ALLOCATION), raster)


@supports_dataset
def direction(raster, x="x", y="y", target_values=[], max_distance=np.inf, distance_metric="EUCLIDEAN"):
    """Compass direction in degrees from every cell to its nearest target (proximity.py:931-1071): 90 east,
    180 south, 270 west, 360 north, 0 on the target itself; NaN beyond `max_distance`."""
    return _wrap(_process(raster, x, y, target_values, max_distance, distance_metric, DIRECTION), raster)

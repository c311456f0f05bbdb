"""xrspatial.convolution on the CUDA backend (reference: convolution.py).

convolve_2d / convolution_2d run on the GPU (xrs_convolve2d_f32); the kernel builders
(circle_kernel, annulus_kernel, custom_kernel, calc_cellsize) are host-side NumPy helpers with
the reference's semantics (convolution.py:30-282).
"""
import ctypes
import re

import numpy as np

from ._xr import DataArray
from .utils import (ArrayTypeFunctionMapping, get_dataarray_resolution, run_stencil_device,
                    run_stencil_host)

DEFAULT_UNIT = 'meter'
UNITS = {'meter': 1, 'meters': 1, 'm': 1,
         'feet': 0.3048, 'foot': 0.3048, 'ft': 0.3048,
         'miles': 1609.344, 'mls': 1609.344, 'ml': 1609.344,
         'kilometer': 1000, 'kilometers': 1000, 'km': 1000}


def _get_distance(distance_str):
    """'<number>[unit]' -> metres (convolution.py:41-75)."""
    parts = [x for x in re.split(r'(-?\d*\.?\d+)', distance_str) if x != '']
    if len(parts) not in (1, 2):
        raise ValueError("Invalid distance.")
    unit = parts[1] if len(parts) == 2 else DEFAULT_UNIT
    try:
        distance = float(parts[0])
    except ValueError:
        raise ValueError("Distance should be a positive numeric value.\n")
    if distance <= 0:
        raise ValueError("Distance should be a positive.\n")
    unit = unit.lower().replace(' ', '')
    if unit not in UNITS:
        raise ValueError(
            "Distance unit should be one of the following: \n"
            "meter (meter, meters, m),\nkilometer (kilometer, kilometers, km),\n"
            "foot (foot, feet, ft),\nmile (mile, miles, ml, mls)")
    return distance * UNITS[unit]


def calc_cellsize(raster):
    """(cellsize_x, |cellsize_y|) in metres, honouring attrs['unit'] (convolution.py:78-132)."""
    unit = raster.attrs.get('unit', DEFAULT_UNIT)
    cellsize_x, cellsize_y = get_dataarray_resolution(raster)
    return cellsize_x * UNITS[unit], np.abs(cellsize_y * UNITS[unit])


def _ellipse_kernel(half_w, half_h):
    x = np.linspace(-half_w, half_w, 2 * half_w + 1)
    y = np.linspace(-half_h, half_h, 2 * half_h + 1)[:, None]
    # inside (x/a)^2 + (y/b)^2 <= 1, written without divisions
    return ((x * half_h) ** 2 + (y * half_w) ** 2 <= (half_w * half_h) ** 2).astype(float)


def circle_kernel(cellsize_x, cellsize_y, radius):
    """0/1 disc of `radius` (number or '<n><unit>') (convolution.py:149-196)."""
    r = _get_distance(str(radius))
    return _ellipse_kernel(int(r / cellsize_x), int(r / cellsize_y))


def annulus_kernel(cellsize_x, cellsize_y, outer_radius, inner_radius):
    """0/1 ring = disc(outer) - centred disc(inner) (convolution.py:199-259)."""
    outer = circle_kernel(cellsize_x, cellsize_y, outer_radius)
    inner = circle_kernel(cellsize_x, cellsize_y, inner_radius)
    pad = np.array(outer.shape) - np.array(inner.shape)
    inner = np.pad(inner, ((pad[0] // 2, pad[0] // 2), (pad[1] // 2, pad[1] // 2)),
                   mode='constant', constant_values=0)
    return outer - inner


def custom_kernel(kernel):
    """Validate a user kernel: ndarray with odd shape (convolution.py:262-282)."""
    if not isinstance(kernel, np.ndarray):
        raise ValueError(
            "Received a custom kernel that is not a Numpy array.",
            "The kernel received was of type {} and needs to be of type `ndarray`".format(type(kernel)))
    rows, cols = kernel.shape
    if rows % 2 == 0 or cols % 2 == 0:
        raise ValueError(
            "Received custom kernel with improper dimensions.",
            "A custom kernel needs to have an odd shape, the supplied kernel "
            "has {} rows and {} columns.".format(rows, cols))
    return kernel


def _kernel_f64(kernel):
    k = np.ascontiguousarray(np.asarray(kernel), dtype=np.float64)
    if k.ndim != 2:
        raise ValueError("kernel must be 2-D")
    return k


def _convolve_2d_numpy(data, kernel):
    """replaces convolution.py:285 `_convolve_2d_numpy` (host raster)."""
    k = _kernel_f64(kernel)
    return run_stencil_host("convolve", data, (k.shape[0], k.shape[1]), aux=k.ravel())


def _convolve_2d_cupy(data, kernel):
    """replaces convolution.py:368 `_convolve_2d_cupy` (device raster)."""
    k = _kernel_f64(kernel)
    return run_stencil_device(data, "xrs_convolve2d_f32", k.ctypes.data_as(ctypes.c_void_p), k.shape[0], k.shape[1])


def convolve_2d(data, kernel):
    """Raw-array correlation of `data` with `kernel` (no flip); float32 result with a NaN ring
    of half the kernel size (convolution.py:389-397)."""
    mapper = ArrayTypeFunctionMapping(numpy_func=_convolve_2d_numpy, cupy_func=_convolve_2d_cupy)
    return mapper(DataArray(data))(data, kernel)


def convolution_2d(agg, kernel, name='convolution_2d'):
    """DataArray wrapper of convolve_2d (convolution.py:400-521)."""
    out = convolve_2d(agg.data, kernel)
    return DataArray(out, name=name, coords=agg.coords, dims=agg.dims, attrs=agg.attrs)

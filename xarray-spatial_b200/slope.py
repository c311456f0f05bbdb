"""xrspatial.slope on the CUDA backend (reference: slope.py:271-371, planar Horn method)."""
from ._xr import DataArray
from .dataset_support import supports_dataset
from .utils import (Z_UNITS, ArrayTypeFunctionMapping, extract_latlon, get_dataarray_resolution,
                    run_geodesic, run_stencil_host, run_surface_device)


def _run_numpy(data, cellsize_x, cellsize_y):
    """Host raster -> xrs_host_stencil(XRS_OP_SLOPE) (replaces slope.py:79 `_run_numpy`)."""
    return run_stencil_host("slope", data, (cellsize_x, cellsize_y))


def _run_cupy(data, cellsize_x, cellsize_y):
    """Device raster -> xrs_slope_f32 (replaces slope.py:145 `_run_cupy`)."""
    return run_surface_device("slope", "xrs_slope_f32", data, cellsize_x, cellsize_y)


@supports_dataset
def slope(agg, name='slope', method='planar', z_unit='meter'):
    """Slope of `agg` in degrees (float32, 1-cell NaN ring).  Same signature and metadata
    contract as the reference; ``method='geodesic'`` fits a plane in the local ECEF tangent frame
    (geodesic.py) and needs lat/lon coordinates on the DataArray."""
    if method not in ('planar', 'geodesic'):
        raise ValueError(f"method must be 'planar' or 'geodesic', got {method!r}")
    if method == 'geodesic':
        if z_unit not in Z_UNITS:
            raise ValueError(f"z_unit must be one of {sorted(set(Z_UNITS.values()), key=str)}, got {z_unit!r}")
        lat, lon, is_2d = extract_latlon(agg)
        out = run_geodesic(agg.data, lat, lon, is_2d, Z_UNITS[z_unit], want_aspect=False)
        return DataArray(out, name=name, coords=agg.coords, dims=agg.dims, attrs=agg.attrs)
    cellsize_x, cellsize_y = get_dataarray_resolution(agg)
    mapper = ArrayTypeFunctionMapping(numpy_func=_run_numpy, cupy_func=_run_cupy)
    out = mapper(agg)(agg.data, cellsize_x, cellsize_y)
    return DataArray(out, name=name, coords=agg.coords, dims=agg.dims, attrs=agg.attrs)

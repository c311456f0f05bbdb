"""xrspatial.aspect on the CUDA backend (reference: aspect.py:274-388, planar)."""
from ._xr import DataArray
from .dataset_support import supports_dataset
from .utils import (Z_UNITS, ArrayTypeFunctionMapping, extract_latlon, run_geodesic, run_stencil_device,
                    run_stencil_host)


def _run_numpy(data):
    """Host raster -> xrs_host_stencil(XRS_OP_ASPECT) (replaces aspect.py:56 `_run_numpy`)."""
    return run_stencil_host("aspect", data)


def _run_cupy(data):
    """replaces aspect.py:139 `_run_cupy`; follows the CPU path (no 359.999 clamp)."""
    return run_stencil_device(data, "xrs_aspect_f32", op="aspect")


@supports_dataset
def aspect(agg, name='aspect', method='planar', z_unit='meter'):
    """Compass aspect in degrees, -1 on flats, NaN ring (float32)."""
    if method not in ('planar', 'geodesic'):
        raise ValueError(f"method must be 'planar' or 'geodesic', got {method!r}")
    if method == 'geodesic':
        if z_unit not in Z_UNITS:
            raise ValueError(f"z_unit must be one of {sorted(set(Z_UNITS.values()), key=str)}, got {z_unit!r}")
        lat, lon, is_2d = extract_latlon(agg)
        out = run_geodesic(agg.data, lat, lon, is_2d, Z_UNITS[z_unit], want_aspect=True)
        return DataArray(out, name=name, coords=agg.coords, dims=agg.dims, attrs=agg.attrs)
    mapper = ArrayTypeFunctionMapping(numpy_func=_run_numpy, cupy_func=_run_cupy)
    out = mapper(agg)(agg.data)
    return DataArray(out, name=name, coords=agg.coords, dims=agg.dims, attrs=agg.attrs)

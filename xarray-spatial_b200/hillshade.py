"""xrspatial.hillshade on the CUDA backend (reference: hillshade.py:103-208, shadows=False)."""
import numpy as np

from ._xr import DataArray
from .dataset_support import supports_dataset
from .utils import is_dask_array, is_device_array, run_stencil_host, run_surface_device


def _run_numpy(data, azimuth=225, angle_altitude=25):
    """replaces hillshade.py:20 `_run_numpy`.  Returns float32 (the dtype the reference
    documents and its GPU path produces; its NumPy path yields float64 only through NumPy-2
    scalar promotion, SURVEY.md 8a row a5)."""
    return run_stencil_host("hillshade", data, (azimuth, angle_altitude))


def _run_cupy(d_data, azimuth, angle_altitude):
    """replaces hillshade.py:78 `_run_cupy`."""
    return run_surface_device("hillshade", "xrs_hillshade_f32", d_data, azimuth, angle_altitude)


@supports_dataset
def hillshade(agg, azimuth=225, angle_altitude=25, name='hillshade', shadows=False):
    """Illumination in [0, 1] from (azimuth, angle_altitude); NaN ring."""
    if shadows:
        raise RuntimeError("Can only calculate shadows if cupy and rtxpy are available")
    if isinstance(agg.data, np.ndarray):
        out = _run_numpy(agg.data, azimuth, angle_altitude)
    elif is_device_array(agg.data):
        out = _run_cupy(agg.data, azimuth, angle_altitude)
    elif is_dask_array(agg.data):
        raise NotImplementedError("dask-backed DataArrays are not supported by the CUDA backend")
    else:
        raise TypeError('Unsupported Array Type: {}'.format(type(agg.data)))
    return DataArray(out, name=name, coords=agg.coords, dims=agg.dims, attrs=agg.attrs)

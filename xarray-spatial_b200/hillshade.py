"""xrspatial.hillshade on the CUDA backend (reference: hillshade.py:103-208, shadows=False)."""
from ._xr import DataArray
from .dataset_support import supports_dataset
from .utils import ArrayTypeFunctionMapping, run_stencil_device, run_stencil_host


def _run_numpy(data, azimuth=225, angle_altitude=25):
    """replaces hillshade.py:20 `_run_numpy`.  Returns float32 (the dtype the reference
    documents and its GPU path produces; its NumPy path yields float64 only through NumPy-2
    scalar promotion, SURVEY.md 8a row a5)."""
    return run_stencil_host("hillshade", data, (azimuth, angle_altitude))


def _run_cupy(d_data, azimuth, angle_altitude):
    """replaces hillshade.py:78 `_run_cupy`."""
    return run_stencil_device(d_data, "xrs_hillshade_f32", azimuth, angle_altitude, op="hillshade")


@supports_dataset
def hillshade(agg, azimuth=225, angle_altitude=25, name='hillshade', shadows=False):
    """Illumination in [0, 1] from (azimuth, angle_altitude); NaN ring."""
    if shadows:
        raise RuntimeError("Can only calculate shadows if cupy and rtxpy are available")
    mapper = ArrayTypeFunctionMapping(numpy_func=_run_numpy, cupy_func=_run_cupy)
    out = mapper(agg)(agg.data, azimuth, angle_altitude)
    return DataArray(out, name=name, coords=agg.coords, dims=agg.dims, attrs=agg.attrs)

"""xrspatial.curvature on the CUDA backend (reference: curvature.py:111-247)."""
from ._xr import DataArray
from .dataset_support import supports_dataset
from .utils import ArrayTypeFunctionMapping, get_dataarray_resolution, run_stencil_device, run_stencil_host


def _run_numpy(data, cellsize):
    """Host raster -> xrs_host_stencil(XRS_OP_CURVATURE) (replaces curvature.py:44 `_run_numpy`)."""
    return run_stencil_host("curvature", data, (cellsize,))


def _run_cupy(data, cellsize):
    """replaces curvature.py:81 `_run_cupy`."""
    return run_stencil_device(data, "xrs_curvature_f32", cellsize, op="curvature")


@supports_dataset
def curvature(agg, name='curvature'):
    """Curvature (-100 * Laplacian / cellsize^2), float32, NaN ring."""
    cellsize_x, cellsize_y = get_dataarray_resolution(agg)
    cellsize = (cellsize_x + cellsize_y) / 2  # curvature.py:234
    mapper = ArrayTypeFunctionMapping(numpy_func=_run_numpy, cupy_func=_run_cupy)
    out = mapper(agg)(agg.data, cellsize)
    return DataArray(out, name=name, coords=agg.coords, dims=agg.dims, attrs=agg.attrs)

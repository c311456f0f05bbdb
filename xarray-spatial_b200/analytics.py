"""xrspatial.analytics.summarize_terrain on the CUDA backend (reference: analytics.py:6-87):
slope + curvature + aspect from ONE pass over the DEM (xrs_surface_suite_f32)."""
import numpy as np

from ._xr import DataArray, Dataset
from .utils import call_on, device_2d, get_dataarray_resolution, is_device_array, pitch, ptr, to_container

_PRODUCTS = ("slope", "aspect", "curvature", "hillshade")   # xrs_surface_suite_f32's outputs, in its order


def surface_suite(agg, azimuth=225, angle_altitude=25, products=_PRODUCTS):
    """dict(product -> DataArray) computed by the fused kernel; device-backed input only
    (host rasters: upload with torch first)."""
    import torch
    data = agg.data
    if not (isinstance(data, np.ndarray) or is_device_array(data)):
        raise TypeError('Unsupported Array Type: {}'.format(type(data)))
    t = device_2d(data, torch.float32)
    csx, csy = get_dataarray_resolution(agg)
    H, W = t.shape
    outs = {p: torch.empty((H, W), dtype=torch.float32, device=t.device) for p in _PRODUCTS if p in products}
    if H and W:
        out_ptrs = [ptr(outs[p]) if p in outs else None for p in _PRODUCTS]
        call_on(t, "xrs_surface_suite_f32", ptr(t), pitch(t), *out_ptrs, W * 4, H, W, float(csx), float(csy),
                float(azimuth), float(angle_altitude))
    return {p: DataArray(to_container(o, data), name=p, coords=agg.coords, dims=agg.dims, attrs=agg.attrs)
            for p, o in outs.items()}


def summarize_terrain(terrain):
    """Dataset with `<name>`, `<name>-slope`, `<name>-curvature`, `<name>-aspect`."""
    if terrain.name is None:
        raise NameError('Requires xr.DataArray.name property to be set')
    res = surface_suite(terrain, products=("slope", "aspect", "curvature"))
    ds = Dataset({terrain.name: terrain}, attrs=terrain.attrs)
    for p in ("slope", "curvature", "aspect"):
        ds[f'{terrain.name}-{p}'] = res[p]          # analytics.py:83-86
    return ds

"""xrspatial.analytics.summarize_terrain on the CUDA backend (reference: analytics.py:6-87):
slope + curvature + aspect from ONE pass over the DEM (xrs_surface_suite_f32)."""
import ctypes

import numpy as np

from . import _lib
from ._xr import DataArray, Dataset
from .utils import device_2d, get_dataarray_resolution, is_device_array, like_container, stream_ptr


def surface_suite(agg, azimuth=225, angle_altitude=25, products=("slope", "aspect", "curvature", "hillshade")):
    """dict(product -> DataArray) computed by the fused kernel; device-backed input only
    (host rasters: upload with torch first)."""
    import torch
    data = agg.data
    if isinstance(data, np.ndarray):
        back = lambda x: x.cpu().numpy()  # noqa: E731
    elif is_device_array(data):
        back = lambda x: like_container(x, data)  # noqa: E731
    else:
        raise TypeError('Unsupported Array Type: {}'.format(type(data)))
    t = device_2d(data, torch.float32)
    csx, csy = get_dataarray_resolution(agg)
    H, W = t.shape
    outs = {}
    ptrs = []
    for p in ("slope", "aspect", "curvature", "hillshade"):
        if p in products:
            outs[p] = torch.empty((H, W), dtype=torch.float32, device=t.device)
            ptrs.append(ctypes.c_void_p(outs[p].data_ptr()))
        else:
            ptrs.append(ctypes.c_void_p(0))
    if H and W:
        with torch.cuda.device(t.device):
            _lib.call("xrs_surface_suite_f32", ctypes.c_void_p(t.data_ptr()), t.stride(0) * 4, *ptrs,
                      W * 4, H, W, float(csx), float(csy), float(azimuth), float(angle_altitude),
                      stream_ptr(t))
    return {p: DataArray(back(o), name=p, coords=agg.coords, dims=agg.dims, attrs=agg.attrs)
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

"""Backend dispatch, resolution and validation helpers -- the L2/L3 layer of the reference
(xrspatial/utils.py) re-stated for the CUDA backend.

Array kinds understood by this package
  * numpy.ndarray            -> "host" runners (xrs_host_* C-ABI, pipelined H2D/compute/D2H)
  * torch CUDA tensor, or any object exposing __cuda_array_interface__ (e.g. cupy.ndarray)
                             -> "device" runners (device-pointer C-ABI on the current stream)
Dask arrays are not supported (the north star excludes Dask): NotImplementedError.
"""
import ctypes
import os

import numpy as np

from . import _lib

try:
    import torch
except ImportError:  # pragma: no cover
    torch = None


def ngjit(f):  # name kept for signature parity; nothing is JIT-compiled in this package
    return f


# ----------------------------------------------------------------------------- array kinds
def is_torch_cuda(a):
    return torch is not None and isinstance(a, torch.Tensor) and a.is_cuda


def is_device_array(a):
    return is_torch_cuda(a) or (hasattr(a, "__cuda_array_interface__") and not isinstance(a, np.ndarray))


def is_dask_array(a):
    return type(a).__module__.split(".")[0] == "dask"


def as_device_tensor(a):
    """View a device array as a torch CUDA tensor (zero copy)."""
    if is_torch_cuda(a):
        return a
    if hasattr(a, "__cuda_array_interface__"):
        return torch.as_tensor(a, device="cuda")
    raise TypeError("not a device array: %r" % type(a))


def like_container(result, template):
    """Return `result` (torch CUDA tensor) in the container type of `template`."""
    if is_torch_cuda(template) or template is None:
        return result
    mod = type(template).__module__.split(".")[0]
    if mod == "cupy":  # pragma: no cover - cupy is optional
        import cupy
        return cupy.asarray(result)
    return result


def stream_ptr(t):
    return ctypes.c_void_p(torch.cuda.current_stream(t.device).cuda_stream)


def host_device_index():
    return int(os.environ.get("XRS_B200_DEVICE", "0"))


def host_devices():
    """CUDA ordinals the host-buffer (numpy) path stripes a raster over.

    XRS_B200_DEVICES = "all" | comma-separated ordinals.  Default: every visible GPU -- one PCIe link
    per stripe -- unless this process is one rank of a one-process-per-GPU job (LOCAL_RANK set, e.g.
    under torchrun) or XRS_B200_DEVICE pins a device, in which case only that GPU is used."""
    spec = os.environ.get("XRS_B200_DEVICES")
    if spec is None:
        if "XRS_B200_DEVICE" in os.environ:
            return [host_device_index()]
        if "LOCAL_RANK" in os.environ:
            return [torch.cuda.current_device() if torch is not None and torch.cuda.is_available()
                    else int(os.environ["LOCAL_RANK"])]
        spec = "all"
    if spec.strip().lower() == "all":
        n = ctypes.c_int(0)
        _lib.call("xrs_device_count", ctypes.byref(n))
        return list(range(max(1, n.value)))
    devs = [int(x) for x in spec.split(",") if x.strip() != ""]
    if not devs or len(set(devs)) != len(devs):
        raise ValueError("XRS_B200_DEVICES must list distinct CUDA ordinals, got %r" % spec)
    return devs


def not_implemented_func(agg, *args, messages='Not yet implemented.'):
    raise NotImplementedError(messages)


class ArrayTypeFunctionMapping(object):
    """utils.py:117-143 with the same constructor; the `cupy_func` slot is the device
    runner and `numpy_func` the host-buffer runner."""

    def __init__(self, numpy_func, cupy_func, dask_func=None, dask_cupy_func=None):
        self.numpy_func = numpy_func
        self.cupy_func = cupy_func
        self.dask_func = dask_func
        self.dask_cupy_func = dask_cupy_func

    def __call__(self, arr):
        data = arr.data
        if isinstance(data, np.ndarray):
            return self.numpy_func
        if is_device_array(data):
            return self.cupy_func
        if is_dask_array(data):
            if self.dask_func is not None:
                return self.dask_func
            raise NotImplementedError("dask-backed DataArrays are not supported by the CUDA backend; "
                                      "row-stripe large rasters with xrspatial_b200.stripes instead")
        raise TypeError("Unsupported Array Type: {}".format(type(arr)))


def validate_arrays(*arrays):
    """utils.py:146-165."""
    if len(arrays) < 2:
        raise ValueError("validate_arrays() input must contain 2 or more arrays")
    first = arrays[0]
    for other in arrays[1:]:
        if not tuple(first.data.shape) == tuple(other.data.shape):
            raise ValueError("input arrays must have equal shapes")
        if not isinstance(first.data, type(other.data)):
            raise ValueError("input arrays must have same type")


# ----------------------------------------------------------------------------- resolution
def get_xy_range(raster, xdim=None, ydim=None):
    if ydim is None:
        ydim = raster.dims[-2]
    if xdim is None:
        xdim = raster.dims[-1]
    xmin = raster[xdim].min().item()
    xmax = raster[xdim].max().item()
    ymin = raster[ydim].min().item()
    ymax = raster[ydim].max().item()
    return (xmin, xmax), (ymin, ymax)


def calc_res(raster, xdim=None, ydim=None):
    """utils.py:204-230."""
    h, w = raster.shape[-2:]
    xrange, yrange = get_xy_range(raster, xdim, ydim)
    xres = (xrange[-1] - xrange[0]) / (w - 1)
    yres = (yrange[-1] - yrange[0]) / (h - 1)
    return xres, yres


def get_dataarray_resolution(agg, xdim=None, ydim=None):
    """utils.py:233-277: attrs['res'] (2-sequence or scalar) else coordinates."""
    try:
        cellsize = agg.attrs.get("res")
        if (isinstance(cellsize, (tuple, np.ndarray, list)) and len(cellsize) == 2
                and isinstance(cellsize[0], (int, float)) and isinstance(cellsize[1], (int, float))):
            cellsize_x, cellsize_y = cellsize
        elif isinstance(cellsize, (int, float)):
            cellsize_x = cellsize
            cellsize_y = cellsize
        else:
            cellsize_x, cellsize_y = calc_res(agg, xdim, ydim)
    except Exception:
        cellsize_x, cellsize_y = calc_res(agg, xdim, ydim)
    return cellsize_x, cellsize_y


# ----------------------------------------------------------------------------- runner helpers
def _dbl_array(vals):
    arr = (ctypes.c_double * max(1, len(vals)))(*[float(v) for v in vals])
    return arr


def device_2d(data, dtype=None):
    """2-D CUDA tensor with unit inner stride and rows at least a row apart, cast to `dtype` when given (like the
    reference's `data.astype(cupy.float32)`, slope.py:150).  A numpy raster is cast on the host and uploaded; a
    device array is viewed, and cast or copied only if needed (a broadcast raster, whose rows share memory, is
    copied)."""
    if isinstance(data, np.ndarray):
        if data.ndim != 2:
            raise ValueError("expected a 2-D raster, got %d-D" % data.ndim)
        np_dtype = None if dtype is None else torch.empty(0, dtype=dtype).numpy().dtype
        return torch.from_numpy(np.ascontiguousarray(data, dtype=np_dtype)).cuda()
    t = as_device_tensor(data)
    if t.dim() != 2:
        raise ValueError("expected a 2-D raster, got %d-D" % t.dim())
    if dtype is not None and t.dtype != dtype:
        t = t.to(dtype)
    if t.numel() and (t.stride(1) != 1 or t.stride(0) < t.shape[1]):
        t = t.clone(memory_format=torch.contiguous_format)   # contiguous() keeps the strides of a 1-row view
    return t


# How each family of device entry points takes a raster's cells (xrs_b200.h names the cell sets):
#   widen: proximity, viewshed, a_star_search and classify read the raster set; other integer and float types are
#          widened to one of it without changing a value;
#   as-is: regions, trim and crop read every zonal cell type as it is;
#   float: perlin and generate_terrain take float32 and float64 only.
# Each policy: (codes of the cell types read, widening, error for another type, its message).
_WIDEN = {"bool": "int16", "int8": "int16", "uint8": "int16", "uint32": "int64", "uint64": "int64",
          "float16": "float32", "bfloat16": "float32"}
CELL_POLICIES = {
    "widen": (_lib.DTYPES, _WIDEN, TypeError, "%s: unsupported cell type %s"),
    "as-is": (_lib.ZONAL_CELLS, {}, NotImplementedError, "%s: %s rasters are not supported (nor by the reference)"),
    "float": ({k: _lib.DTYPES[k] for k in ("float32", "float64")}, {}, TypeError,
              "%s takes float32 or float64 cells, not %s"),
}


def raster_cells(data, what, policy):
    """A numpy or device 2-D raster checked against CELL_POLICIES[policy], as the numpy array or CUDA tensor of the
    cells the entry point reads, and their code.  Nothing is uploaded."""
    if is_dask_array(data):
        raise NotImplementedError("%s: Dask arrays are not supported by the GPU backend" % what)
    if isinstance(data, np.ndarray):
        a = data
    elif is_device_array(data):
        a = as_device_tensor(data)
    else:
        raise TypeError("Unsupported raster array type: {}".format(type(data)))
    if a.ndim != 2:
        raise ValueError("%s needs a 2-D raster, got %d-D" % (what, a.ndim))
    codes, widen, error, message = CELL_POLICIES[policy]
    name = str(a.dtype).replace("torch.", "")
    host = isinstance(a, np.ndarray)
    if name == "uint64" and widen.get(name) == "int64":
        # uint64 cells below 2**63 are their own int64 view; the others are the negative ones of it
        a, name = a.view(np.int64 if host else torch.int64), "int64"
        if bool((a < 0).any()):
            raise ValueError("%s: uint64 cells above 2**63 - 1 are not supported" % what)
    elif name in widen:
        name = widen[name]
        a = a.astype(name) if host else a.to(getattr(torch, name))
    if name not in codes:
        raise error(message % (what, name))
    return a, codes[name]


def device_cells(data, what, policy):
    """raster_cells on the device: (a 2-D CUDA tensor as device_2d gives it, the cells' code)."""
    a, code = raster_cells(data, what, policy)
    return device_2d(a), code


def device_scratch(query, *query_args, device, what):
    """(a device buffer of the bytes `query(*query_args)` asks for, that size).  MemoryError when the device
    cannot allocate it."""
    need = ctypes.c_int64()
    _lib.call(query, *query_args, ctypes.byref(need))
    try:
        return torch.empty(max(1, need.value), dtype=torch.uint8, device=device), need.value
    except torch.OutOfMemoryError as e:
        raise MemoryError("%s needs %d bytes of device scratch" % (what, need.value)) from e


def ptr(t):
    return ctypes.c_void_p(t.data_ptr())


def pitch(t):
    """Bytes between the rows of a 2-D tensor."""
    return t.stride(0) * t.element_size()


def call_on(t, name, *args):
    """The entry point `name(*args, stream)` on tensor t's device, on torch's current stream there."""
    with torch.cuda.device(t.device):
        _lib.call(name, *args, stream_ptr(t))


def to_container(out, data):
    """A device result `out` in the container of the raster `data`: numpy for numpy, else like_container."""
    return out.cpu().numpy() if isinstance(data, np.ndarray) else like_container(out, data)


def coord(raster, name):
    """raster[name] as a numpy array (the integer index when the raster has no such coordinate)."""
    c = raster[name]
    return np.asarray(getattr(c, "data", c))


def run_stencil_device(fn_name, data, *args, dtype=None):
    """Call the device entry point `fn_name(in, in_pitch, out, out_pitch, H, W, *args, stream)` on
    torch's current stream, `args` being its own arguments in header order.  The raster is cast to
    `dtype` (default float32) and the result has the same dtype."""
    t = device_2d(data, dtype or torch.float32)
    H, W = t.shape
    out = torch.empty((H, W), dtype=t.dtype, device=t.device)
    if H == 0 or W == 0:
        return like_container(out, data)
    esz = t.element_size()
    with torch.cuda.device(t.device):
        _lib.call(fn_name, ctypes.c_void_p(t.data_ptr()), t.stride(0) * esz, ctypes.c_void_p(out.data_ptr()),
                  out.stride(0) * esz, H, W, *args, stream_ptr(t))
    return like_container(out, data)


_SURFACE_OPS = ("slope", "aspect", "curvature", "hillshade")
_SURFACE_CELLS = ("int16", "uint16", "int32", "float64")   # what the direct-ingest kernels read


def run_surface_device(op, fn_name, data, *scalars):
    """slope / aspect / curvature / hillshade on a device raster.  int16 / uint16 / int32 / float64
    rasters go through the direct-ingest kernels (xrs_surface_typed: no separate cast pass); other
    dtypes are cast to float32 first, like the reference does (slope.py:150)."""
    t = as_device_tensor(data)
    cells = str(t.dtype).replace("torch.", "")
    if cells in _SURFACE_CELLS and t.dim() == 2 and t.numel() and t.stride(1) == 1:
        H, W = t.shape
        out = torch.empty((H, W), dtype=torch.float32, device=t.device)
        try:
            with torch.cuda.device(t.device):
                _lib.call("xrs_surface_typed", _lib.OPS[op], ctypes.c_void_p(t.data_ptr()), _lib.DTYPES[cells],
                          t.stride(0) * t.element_size(), ctypes.c_void_p(out.data_ptr()), out.stride(0) * 4, H, W,
                          _dbl_array(scalars), stream_ptr(t))
            return like_container(out, data)
        except NotImplementedError:
            pass  # layout the ingest kernels do not take (odd width, misaligned rows): cast instead
    return run_stencil_device(fn_name, data, *[float(s) for s in scalars])


def run_stencil_host(op, data, p=(), aux=()):
    """xrs_host_stencil on a numpy raster over host_devices(); the result is a numpy array in pinned
    memory.  The cells that cross PCIe follow the C entry point's table:
      * slope / aspect / curvature / hillshade: int16, uint16, int32 and float64 rasters as they are
        when W % 4 == 0 (converted on the device; half the bytes for 16-bit DEMs), anything else cast
        to float32 (slope.py:58); float32 result;
      * focal mean: float32 as it is, anything else cast to float64; float64 result (focal.py:257);
      * convolve / focal statistics: cast to float32; float32 result."""
    from . import _hostmem
    if data.ndim != 2:
        raise ValueError("expected a 2-D raster, got %d-D" % data.ndim)
    H, W = data.shape
    cells, out_dtype = "float32", np.float32
    if op == "focal_mean":
        cells, out_dtype = ("float32" if data.dtype.name == "float32" else "float64"), np.float64
    elif op in _SURFACE_OPS and data.dtype.name in _SURFACE_CELLS and W % 4 == 0:
        cells = data.dtype.name
    if H == 0 or W == 0:
        return np.empty((H, W), out_dtype)
    d = np.ascontiguousarray(data, dtype=cells)
    out = _hostmem.empty((H, W), out_dtype)
    devs = host_devices()
    _lib.call("xrs_host_stencil", _lib.OPS[op], ctypes.c_void_p(d.ctypes.data), _lib.DTYPES[cells],
              ctypes.c_void_p(out.ctypes.data), H, W, _dbl_array(p), _dbl_array(aux), len(aux),
              (ctypes.c_int * len(devs))(*devs), len(devs))
    return out


# ----------------------------------------------------------------------------- geodesic helpers
# z-unit factors and lat/lon extraction for method='geodesic' (utils.py:593-713)
Z_UNITS = {
    'meter': 1.0, 'meters': 1.0, 'm': 1.0,
    'foot': 0.3048, 'feet': 0.3048, 'ft': 0.3048,
    'kilometer': 1000.0, 'kilometers': 1000.0, 'km': 1000.0,
    'mile': 1609.344, 'miles': 1609.344, 'mi': 1609.344,
}
_LAT_NAMES = {'lat', 'latitude', 'y'}
_LON_NAMES = {'lon', 'longitude', 'x'}


def _coord_values(agg, name):
    c = agg.coords[name]
    return np.asarray(getattr(c, "values", c))


def _find_coord(agg, dim_name, known_names, label):
    """A numeric coordinate named like the dimension, else any coordinate with a known name."""
    if dim_name in agg.coords and np.issubdtype(_coord_values(agg, dim_name).dtype, np.number):
        return _coord_values(agg, dim_name)
    for name in agg.coords:
        if str(name).lower() in known_names and np.issubdtype(_coord_values(agg, name).dtype, np.number):
            return _coord_values(agg, name)
    raise ValueError(
        f"geodesic method requires {label} coordinates on the DataArray. "
        f"No numeric coordinate found for dim '{dim_name}' or any of {sorted(known_names)}.")


def _validate_geographic_range(lat, lon):
    lat_min, lat_max = np.nanmin(lat), np.nanmax(lat)
    lon_min, lon_max = np.nanmin(lon), np.nanmax(lon)
    if lat_min < -90 or lat_max > 90:
        raise ValueError(f"Latitude values must be in [-90, 90], got [{lat_min}, {lat_max}]. "
                         f"Are your coordinates in a projected CRS?")
    if lon_min < -180 or lon_max > 360:
        raise ValueError(f"Longitude values must be in [-180, 360], got [{lon_min}, {lon_max}]. "
                         f"Are your coordinates in a projected CRS?")
    if lat_max - lat_min > 180 or lon_max - lon_min > 360:
        raise ValueError(f"Coordinate span too large for geographic coordinates "
                         f"(lat span={lat_max - lat_min}, lon span={lon_max - lon_min}). "
                         f"Are your coordinates in a projected CRS?")


def extract_latlon(agg):
    """(lat, lon, is_2d): float64 latitude / longitude of the raster's cells -- 1-D per-row /
    per-column vectors for a regular grid, (H, W) arrays for a curvilinear one (utils.py:608-662,
    without materialising the broadcast for regular grids)."""
    if agg.ndim < 2:
        raise ValueError(f"geodesic method requires a 2-D DataArray, got {agg.ndim}-D")
    dim_y, dim_x = agg.dims[-2], agg.dims[-1]
    lat = np.asarray(_find_coord(agg, dim_y, _LAT_NAMES, 'latitude'), dtype=np.float64)
    lon = np.asarray(_find_coord(agg, dim_x, _LON_NAMES, 'longitude'), dtype=np.float64)
    if lat.ndim == 1 and lon.ndim == 1:
        is_2d = False
    elif lat.ndim == 2 and lon.ndim == 2:
        is_2d = True
    else:
        raise ValueError(f"lat/lon coordinates must be both 1-D or both 2-D, got lat={lat.ndim}-D and lon={lon.ndim}-D")
    _validate_geographic_range(lat, lon)
    return np.ascontiguousarray(lat), np.ascontiguousarray(lon), is_2d


def run_geodesic(data, lat, lon, is_2d, z_factor, want_aspect):
    """xrs_geodesic on a device or host raster; result in the container type of `data`."""
    t = device_2d(data)
    if t.dtype not in (torch.float32, torch.float64):
        t = t.to(torch.float64)           # the reference computes on data.astype(float64), slope.py:169
    H, W = t.shape
    out = torch.empty((H, W), dtype=torch.float32, device=t.device)
    if H and W:
        lat_t = torch.as_tensor(lat, dtype=torch.float64, device=t.device).contiguous()
        lon_t = torch.as_tensor(lon, dtype=torch.float64, device=t.device).contiguous()
        with torch.cuda.device(t.device):
            _lib.call("xrs_geodesic", ctypes.c_void_p(t.data_ptr()), 0 if t.dtype == torch.float32 else 1,
                      t.stride(0) * t.element_size(), ctypes.c_void_p(lat_t.data_ptr()),
                      ctypes.c_void_p(lon_t.data_ptr()), 1 if is_2d else 0, ctypes.c_void_p(out.data_ptr()),
                      out.stride(0) * 4, H, W, float(z_factor), 1 if want_aspect else 0, stream_ptr(t))
    if isinstance(data, np.ndarray):
        return out.cpu().numpy()
    return like_container(out, data)

"""perlin (perlin.py:189 of the reference) on the GPU, and the noise runner generate_terrain shares.

The semantics are the reference's NumPy path (_perlin_numpy, _terrain_numpy), bit for bit where NumPy's own
arithmetic is (DESIGN.md section 4.10): the permutation tables are RandomState(seed).permutation(2**20), built on
the device; the coordinates are NumPy's float32 linspace, built on the host; each octave is evaluated in float64
without contraction, in the order numba evaluates it.

Documented deviations from the reference:
  1. The input is never written (the reference's perlin writes its result into the caller's buffer and returns
     that buffer).
  2. NumPy's global generator is not reseeded.
  3. Cell types other than float32 and float64 raise TypeError (the reference writes truncated values for integer
     cells and computes float16 in half precision).
  4. Device containers get the NumPy path's result; the reference's cupy kernel is fastmath with float64
     coordinates, and the reference's own tests allow it rtol=1e-5 against NumPy.
"""
import ctypes
import operator

import numpy as np

from ._xr import DataArray
from .utils import call_on, device_2d, device_scratch, host_device_index, is_dask_array, ptr, raster_cells
from .utils import to_container

TABLE_N = 2 ** 20          # the reference's permutation(2**20)
INDEX_LIMIT = 2 ** 21      # np.append(p, p) takes indices in [-2**21, 2**21)
TERRAIN_OCTAVES = 16


def check_seed(seed, count=1):
    """The seeds seed .. seed + count - 1 as ints, with np.random.seed's rule: each must lie in [0, 2**32 - 1]."""
    try:
        s = operator.index(seed)
    except TypeError:
        raise TypeError("Cannot cast seed of type %s to an integer" % type(seed).__name__) from None
    if s < 0 or s + count - 1 > 2 ** 32 - 1:
        raise ValueError("Seed must be between 0 and 2**32 - 1")
    return [s + k for k in range(count)]


def check_cells(data, fname):
    """A numpy or device raster of float32 / float64 cells with at least one cell."""
    if 0 in raster_cells(data, fname, "float")[0].shape:
        raise ValueError("zero-size array to reduction operation minimum which has no identity")


def perm_tables(seeds, device, rounds=None):
    """RandomState(s).permutation(2**20) for each seed, as one (len(seeds), 2**20) int32 tensor on `device`, built
    there on torch's current stream."""
    import torch
    n = TABLE_N
    tables = torch.empty((len(seeds), n), dtype=torch.int32, device=device)
    scratch, size = device_scratch("xrs_perm_tables_scratch_bytes", len(seeds), n, device=device,
                                   what="the permutation tables")
    host = (ctypes.c_uint32 * len(seeds))(*seeds)
    r = ctypes.c_int64()
    call_on(tables, "xrs_perm_tables", ctypes.cast(host, ctypes.c_void_p), len(seeds), n, ptr(tables), ptr(scratch),
            size, ctypes.byref(r))
    if rounds is not None:
        rounds.append(r.value)
    return tables


def index_out_of_range(stats):
    """Whether the reference indexes its doubled table outside [-2**21, 2**21) somewhere: a column's xi or xi + 1
    outside it, a row's yi beyond 2**22, or P[xi] + yi (+ 1) outside it for some column and row.  `stats` holds,
    per octave, the bad-coordinate flag, the least and largest of P[xi], P[xi + 1] and the least and largest yi."""
    for bad, pmin, pmax, ymin, ymax in np.asarray(stats).reshape(-1, 5).tolist():
        if bad or pmin + ymin < -INDEX_LIMIT or pmax + ymax + 1 >= INDEX_LIMIT:
            return True
    return False


def run_noise(data, seeds, xs, ys, terrain, zfactor=0.0):
    """The noise field of a checked raster (check_cells) in its container: perlin (terrain False, one seed) or
    generate_terrain's array (16 seeds).  xs, ys: the float32 coordinates of the columns and rows."""
    import torch
    if isinstance(data, np.ndarray):
        device = torch.device("cuda", host_device_index())
        t = torch.from_numpy(np.ascontiguousarray(data)).to(device) if terrain else None
    else:
        t = device_2d(data)
        device = t.device
    H, W = data.shape
    dtype = torch.float32 if str(data.dtype).endswith("float32") else torch.float64
    code = 0 if dtype == torch.float32 else 1
    with torch.cuda.device(device):
        tables = perm_tables(seeds, device)
        dx = torch.from_numpy(np.ascontiguousarray(xs, dtype=np.float32)).to(device)
        dy = torch.from_numpy(np.ascontiguousarray(ys, dtype=np.float32)).to(device)
        scratch, size = device_scratch("xrs_noise_scratch_bytes", H, W, int(terrain), device=device,
                                       what="the noise of a %d x %d raster" % (H, W))
        try:
            out = torch.empty((H, W), dtype=dtype, device=device)
        except torch.OutOfMemoryError as e:
            raise MemoryError("the noise of a %d x %d raster needs %d bytes of device memory"
                              % (H, W, H * W * (4 if code == 0 else 8))) from e
        stats = torch.empty((len(seeds), 5), dtype=torch.int32, device=device)
        esz = out.element_size()
        call_on(out, "xrs_noise", ptr(t) if t is not None else None, code, t.stride(0) * esz if t is not None else 0,
                H, W, ptr(tables), ptr(dx), ptr(dy), int(terrain), float(zfactor), ptr(out), out.stride(0) * esz,
                ptr(stats), ptr(scratch), size)
        if index_out_of_range(stats.cpu().numpy()):
            raise IndexError("index out of bounds for the permutation table of size %d" % INDEX_LIMIT)
    return to_container(out, data)


def perlin(agg, freq=(1, 1), seed=5, name='perlin'):
    """Perlin noise over the cells of `agg`, normalised to [0, 1]: the reference's NumPy result, on the GPU.

    `freq` is the (x, y) frequency: column j sits at x = linspace(0, freq[0], W, endpoint=False) in float32, row i
    at y likewise.  The gradients come from RandomState(seed).permutation(2**20).  Same cell type and container
    out as in (float32 or float64), with the input's dims and attrs and no coords; NaN everywhere when every cell
    has the same noise (a 1 x 1 raster).  The input is not written.  IndexError where the reference raises it
    (coordinates beyond the doubled permutation table); ValueError for a seed outside [0, 2**32 - 1], an empty or
    non-2-D raster; TypeError for other cell types; NotImplementedError for Dask arrays."""
    data = agg.data
    if is_dask_array(data):
        raise NotImplementedError("perlin: Dask arrays are not supported by the GPU backend")
    seeds = check_seed(seed)
    check_cells(data, "perlin")
    H, W = data.shape
    xs = np.linspace(0, freq[0], W, endpoint=False, dtype=np.float32)
    ys = np.linspace(0, freq[1], H, endpoint=False, dtype=np.float32)
    out = run_noise(data, seeds, xs, ys, terrain=False)
    return DataArray(out, dims=agg.dims, attrs=agg.attrs, name=name)

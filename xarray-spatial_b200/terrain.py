"""generate_terrain (terrain.py:183 of the reference) on the GPU.

The array is the reference's NumPy path (_terrain_numpy): 16 octaves of the perlin noise, octave o from
RandomState(seed + o).permutation(2**20) at float32(x 2^o) weighed by 2^-o, summed into the input times 0 in its
cell type, divided by 1.97, cubed, normalised, cells below 0.3 set to 0 and multiplied by zfactor (DESIGN.md
section 4.10).  Every step but the cube is NumPy's arithmetic bit for bit.  NumPy's float32 power is not correctly
rounded; here the float32 cube is rounded once from the float64 product, and the float64 cube is h h h.  The
deviations of perlin (perlin.py) apply: the input is not written, NumPy's global generator is not reseeded, cell
types other than float32 and float64 raise TypeError, and device containers get the NumPy path's result.
"""
import numpy as np

from ._xr import DataArray, ShimDataArray
from .perlin import TERRAIN_OCTAVES, check_cells, check_seed, run_noise
from .utils import get_dataarray_resolution, is_dask_array


def _scale(value, old_range, new_range):
    d = (value - old_range[0]) / (old_range[1] - old_range[0])
    return d * (new_range[1] - new_range[0]) + new_range[0]


def _pixel_centres(rng, n):
    """The coordinates datashader's Canvas gives n pixels over `rng` (its LinearAxis): s = n / (end - start),
    t = -start s, coordinate j = (j + 0.5 - t) / s.  Restated from datashader's source; datashader itself is not
    a dependency, so this is not checked against it."""
    start, end = rng
    s = n / (end - start)
    t = -start * s
    return (np.arange(n) + 0.5 - t) / s


def generate_terrain(agg, x_range=(0, 500), y_range=(0, 500), seed=10, zfactor=4000, full_extent=None,
                     name='terrain'):
    """Pseudo-random terrain over the cells of `agg`: the reference's NumPy result, on the GPU.

    `x_range` and `y_range` place the raster within `full_extent` (xmin, ymin, xmax, ymax; default the ranges
    themselves), which maps to the noise's unit square.  Same cell type (float32 or float64) and container out as
    in, dims ('y', 'x'), the pixel-centre coordinates datashader's Canvas gives those ranges (y ascending),
    attrs {'res': ...} and `name`.  Every cell is NaN when a cell of `agg` is NaN or infinite.  The input is not
    written.  IndexError where the reference raises it; ValueError for a seed + 15 outside [0, 2**32 - 1] or an
    empty or non-2-D raster; ZeroDivisionError for a zero-width extent; TypeError for other cell types;
    NotImplementedError for Dask arrays."""
    height, width = agg.shape

    if full_extent is None:
        full_extent = (x_range[0], y_range[0],
                       x_range[1], y_range[1])

    elif not isinstance(full_extent, (list, tuple)) and len(full_extent) != 4:
        raise TypeError('full_extent must be tuple(4)')

    full_xrange = (full_extent[0], full_extent[2])
    full_yrange = (full_extent[1], full_extent[3])

    x_range_scaled = (_scale(x_range[0], full_xrange, (0.0, 1.0)),
                      _scale(x_range[1], full_xrange, (0.0, 1.0)))

    y_range_scaled = (_scale(y_range[0], full_yrange, (0.0, 1.0)),
                      _scale(y_range[1], full_yrange, (0.0, 1.0)))

    data = agg.data
    if is_dask_array(data):
        raise NotImplementedError("generate_terrain: Dask arrays are not supported by the GPU backend")
    seeds = check_seed(seed, TERRAIN_OCTAVES)
    check_cells(data, "generate_terrain")
    xs = np.linspace(x_range_scaled[0], x_range_scaled[1], width, endpoint=False, dtype=np.float32)
    ys = np.linspace(y_range_scaled[0], y_range_scaled[1], height, endpoint=False, dtype=np.float32)
    out = run_noise(data, seeds, xs, ys, terrain=True, zfactor=zfactor)

    coords = {"y": _pixel_centres(y_range, height), "x": _pixel_centres(x_range, width)}
    grid = ShimDataArray(np.broadcast_to(np.float32(0), (height, width)), coords=coords, dims=("y", "x"))
    res = get_dataarray_resolution(grid)
    return DataArray(out, name=name, coords=coords, dims=("y", "x"), attrs={"res": res})

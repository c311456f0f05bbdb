"""a_star_search (pathfinding.py:233-382 of the reference) on the GPU.

The search returns a shortest path over the crossable cells, exactly: path lengths are kept as counts of
orthogonal and diagonal steps and compared in integers (DESIGN.md section 4.9).  A tiled relaxation builds the
field of shortest lengths to the goal, and a walk from the start follows it, taking at each cell the first move of
the reference's neighbour order that stays on a shortest path.

What is guaranteed against the reference: the same reachability, the same path length in orthogonal and diagonal
steps, path values that are the running sums along the returned path, and the reference's array wherever the
shortest path is unique.  Among several equally short paths the reference returns the one its pop order finds,
which a parallel search cannot reproduce; this one returns the path the rule above picks.  For very long paths the
reference's float64 comparisons could accept a path whose exact length exceeds the shortest by less than their
rounding error; this implementation never does.
"""
import ctypes
import warnings

import numpy as np

from . import _lib
from ._xr import DataArray
from .utils import as_device_tensor, call_on, coord, device_cells, device_scratch, get_dataarray_resolution
from .utils import is_dask_array, is_device_array, pitch, ptr, to_container

NONE = -1


def _get_pixel_id(point, raster, xdim, ydim):
    """The (row, column) of a (y, x) point: int(|p - coord[0]| / cellsize) along each axis."""
    cellsize_x, cellsize_y = get_dataarray_resolution(raster, xdim, ydim)
    py = int(abs(point[0] - coord(raster, ydim)[0]) / cellsize_y)
    px = int(abs(point[1] - coord(raster, xdim)[0]) / cellsize_x)
    return py, px


def _is_inside(py, px, h, w):
    return 0 <= px < w and 0 <= py < h


def _barrier_values(barriers):
    """The barriers as float64, as the reference compares them with the cells, without NaN (it matches nothing)."""
    b = np.asarray(barriers, dtype=np.float64).ravel()
    return b[~np.isnan(b)]


def _crossable_rule(bars):
    """crossable(v): the reference's _is_not_crossable negated, for a cell value v widened to float64."""
    return lambda v: not (np.isnan(v) or np.any(v == bars))


def _plan(surface, start, goal, barriers, x, y, connectivity, snap_start, snap_goal, cell, snap):
    """a_star_search's glue (pathfinding.py:327-375): the argument checks, the start and goal cells, the snaps
    and the warnings.  `cell(row, col)` returns a cell as a float64 (row, col may be -1, -1: the last cell, as the
    reference reads it); `snap(row, col)` is the snap of a non-crossable cell.  Returns the barriers as float64
    and the start and goal cells, or None when the output is all NaN."""
    if surface.ndim != 2:
        raise ValueError("input `surface` must be 2D")
    if tuple(surface.dims) != (y, x):
        raise ValueError("`surface.coords` should be named as coordinates:({}, {})".format(y, x))
    if connectivity != 4 and connectivity != 8:
        raise ValueError("Use either 4 or 8-connectivity.")
    start_py, start_px = _get_pixel_id(start, surface, x, y)
    goal_py, goal_px = _get_pixel_id(goal, surface, x, y)
    h, w = surface.shape
    if not _is_inside(start_py, start_px, h, w):
        raise ValueError("start location outside the surface graph.")
    if not _is_inside(goal_py, goal_px, h, w):
        raise ValueError("goal location outside the surface graph.")
    bars = _barrier_values(barriers)
    crossable = _crossable_rule(bars)
    if snap_start and not crossable(cell(start_py, start_px)):
        start_py, start_px = snap(bars, start_py, start_px)
    start_ok = crossable(cell(start_py, start_px))
    if not start_ok:
        warnings.warn("Start at a non crossable location", Warning)
    if snap_goal and not crossable(cell(goal_py, goal_px)):
        goal_py, goal_px = snap(bars, goal_py, goal_px)
    goal_ok = crossable(cell(goal_py, goal_px))
    if not goal_ok:
        warnings.warn("End at a non crossable location", Warning)
    run = start_py != NONE and goal_py != NONE and start_ok and goal_ok
    return bars, ((start_py, start_px), (goal_py, goal_px)) if run else None


def a_star_search(surface, start, goal, barriers=[], x="x", y="y", connectivity=8, snap_start=False,
                  snap_goal=False):
    """Shortest path from `start` to `goal`, both (y, x) coordinates, through the crossable cells of `surface`.

    A cell is crossable unless it is NaN or equal to one of `barriers`; a move goes to one of the 8 neighbours (4
    with `connectivity=4`) and costs its pixel-space length, 1 or sqrt(2).  `snap_start` / `snap_goal` move a
    non-crossable start or goal to the nearest crossable cell.  float64 result with the input's coords, dims and
    attrs: NaN except along the path, whose cells hold the length walked from the start (0 there); all NaN when
    there is no path.  Of several shortest paths, the one taken leaves each cell by the first move of the
    reference's neighbour order that stays on a shortest path."""
    import torch
    data = surface.data
    if is_dask_array(data):
        raise NotImplementedError("a_star_search: Dask arrays are not supported by the GPU backend")
    if not (isinstance(data, np.ndarray) or is_device_array(data)):
        raise TypeError("Unsupported raster array type: {}".format(type(data)))
    dev = {}

    def cells(bars):   # the raster on the device and the C arguments that describe it and the barriers
        if "t" not in dev:
            dev["t"], code = device_cells(data, "a_star_search", "widen")
            t = dev["t"]
            dev["bars"] = torch.as_tensor(np.append(bars, 0.0), device=t.device)   # never a NULL pointer
            dev["args"] = (ptr(t), code, pitch(t), t.shape[0], t.shape[1], ptr(dev["bars"]), bars.size)
        return dev["t"], dev["args"]

    def cell(py, px):
        if isinstance(data, np.ndarray):
            return float(data[py, px])
        return float(as_device_tensor(data)[py, px].item())

    def snap(bars, py, px):
        t, args = cells(bars)
        r, c = ctypes.c_int64(), ctypes.c_int64()
        scratch = torch.empty(256, dtype=torch.uint8, device=t.device)
        call_on(t, "xrs_a_star_snap", *args, py, px, ctypes.byref(r), ctypes.byref(c), ptr(scratch), 256)
        return r.value, c.value

    bars, cells_of_path = _plan(surface, start, goal, barriers, x, y, connectivity, snap_start, snap_goal, cell,
                                snap)
    t, args = cells(bars)
    H, W = t.shape
    if cells_of_path is None:
        _lib.call("xrs_a_star_scratch_bytes", H, W, ctypes.byref(ctypes.c_int64()))   # the raster's size limit
        out = torch.full((H, W), float("nan"), dtype=torch.float64, device=t.device)
    else:
        (sr, sc), (gr, gc) = cells_of_path
        scratch, size = device_scratch("xrs_a_star_scratch_bytes", H, W, device=t.device, what="a_star_search")
        out = torch.empty((H, W), dtype=torch.float64, device=t.device)
        call_on(t, "xrs_a_star_search", *args, connectivity, sr, sc, gr, gc, ptr(out), pitch(out), ptr(scratch),
                size, None)
    return DataArray(to_container(out, data), coords=surface.coords, dims=surface.dims, attrs=surface.attrs)

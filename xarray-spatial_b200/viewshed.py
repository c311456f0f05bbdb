"""viewshed (viewshed.py:1505-1675 of the reference) on the GPU.

The reference sweeps every cell's events around the observer through a red-black tree (a port of GRASS
r.viewshed).  Here each cell decides on its own with the same test the sweep makes for it, so the visible /
invisible decision and the vertical angles are the reference's (DESIGN.md section 4.8).

One deviation: the reference raises ValueError("node not found") when a NaN cell lies in the observer's row east
of the observer.  This implementation returns the well-defined result instead: NaN cells are -1 (invisible) and
never block the view of other cells, as everywhere else in the raster.
"""
import numpy as np

from ._xr import DataArray
from .utils import call_on, coord, device_2d, device_scratch, pitch, ptr, raster_cells, to_container

OBS_ELEV = 0
TARGET_ELEV = 0


def _nearest(coords, v):
    """The index xarray's sel(method='nearest') picks: the nearest coordinate, the larger value on a tie, and of
    equal coordinates the first."""
    d = np.abs(coords - v)
    best = coords[d == d.min()].max()
    return int(np.flatnonzero(coords == best)[0])


def _view(xs, ys, x, y, z_at, observer_elev, target_elev):
    """_viewshed_cpu's glue: the observer cell (row, column), its elevation, the target offset and the
    resolutions.  `z_at(row, col)` returns the raster's cell as a NumPy scalar of its own type."""
    if not (xs.min() <= x <= xs.max()):
        raise ValueError("x argument outside of raster x_range")
    if not (ys.min() <= y <= ys.max()):
        raise ValueError("y argument outside of raster y_range")
    vc, vr = _nearest(xs, x), _nearest(ys, y)
    vp_elev = float(z_at(vr, vc) + observer_elev)   # in the raster's own type first, as NumPy adds them
    target = float(target_elev) if abs(target_elev) > 0 else 0.0
    with np.errstate(divide="ignore", invalid="ignore"):   # one row or column: NaN, as in the reference
        ew_res = float((xs[-1] - xs[0]) / (len(xs) - 1))
        ns_res = float((ys[-1] - ys[0]) / (len(ys) - 1))
    return vr, vc, vp_elev, target, ew_res, ns_res


def viewshed(raster, x, y, observer_elev=OBS_ELEV, target_elev=TARGET_ELEV):
    """Cells visible from an observer standing `observer_elev` above the cell nearest to (x, y).

    float64 result with the input's coords, dims and attrs: 180 at the observer, the vertical angle in degrees
    of every visible cell (0 straight below the observer, 90 level, 180 straight above), -1 elsewhere.
    `target_elev` is added to every cell seen as a target.  NaN cells are -1 and never block (the reference
    raises when one lies in the observer's row east of it)."""
    import torch
    data = raster.data
    cells, code = raster_cells(data, "viewshed", "widen")
    xs, ys = coord(raster, "x"), coord(raster, "y")
    if (len(xs), len(ys)) != tuple(cells.shape[::-1]):
        raise ValueError("coordinate lengths (%d, %d) do not match the raster's shape %s"
                         % (len(ys), len(xs), tuple(cells.shape)))
    if isinstance(data, np.ndarray):
        view = _view(xs, ys, x, y, lambda r, c: data[r, c], observer_elev, target_elev)
    else:
        view = _view(xs, ys, x, y, lambda r, c: cells[r, c].cpu().numpy()[()], observer_elev, target_elev)
    t = device_2d(cells)
    vr, vc, vp_elev, target, ew_res, ns_res = view
    H, W = t.shape
    scratch, size = device_scratch("xrs_viewshed_scratch_bytes", H, W, device=t.device, what="viewshed")
    out = torch.empty((H, W), dtype=torch.float64, device=t.device)
    call_on(t, "xrs_viewshed", ptr(t), code, pitch(t), H, W, vr, vc, vp_elev, target, ew_res,
            ns_res, ptr(out), pitch(out), ptr(scratch), size)
    return DataArray(to_container(out, data), coords=raster.coords, dims=raster.dims, attrs=raster.attrs)

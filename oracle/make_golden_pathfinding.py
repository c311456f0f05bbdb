"""Generate tests/golden/pathfinding_reference.npz and pathfinding_signature.json from the UNMODIFIED reference.

TEST INFRASTRUCTURE (needs a checkout of the reference, like make_golden.py; the existing golden files are not
touched).  Every output comes from the reference's public `a_star_search` (pathfinding.py:233-382): the pixel
mapping through get_dataarray_resolution, the snapping, the warnings and the A* loop.  ref_loader's stub DataArray
has no coordinate lookup, so a small adapter supplies `raster[name].min().item()` and the coords' `.data`.

Every case is one call: rows of int64 or float64 cells, y coordinates descending from (H - 1) ry to 0 and x
ascending from 0 to (W - 1) rx (the reference tests' create_test_raster layout), `attrs['res'] = (rx, ry)` or no
attrs (the resolution then comes from the coordinates), a barrier list, (y, x) start and goal points,
connectivity and snap flags.  Stored with each case: the output, the warnings raised, the reference path's exact
step counts (a orthogonal, b diagonal; -1 without a path) and `unique`, whether the shortest path is the only one
(counted over the exact graph).

* `doc`, `fix8`, `fix4`: the docstring example and the reference test_pathfinding.py connectivity fixtures;
  `nobar`: test_a_star_search_no_barriers's loops (every start and goal) on its fixture, stored as small cases.
* `small_*`: ~400 seeded rasters of 2-40 cells a side, concatenated (offsets in `small_off`).
* `large_*`: rasters of 200-400 cells a side -- random obstacles, a serpentine maze and a DEM with NaN water;
  the cells are stored packed and the output as the path's row-major indices and values.

Usage:  XRS_REFERENCE_ROOT=<reference checkout> python oracle/make_golden_pathfinding.py
"""
import heapq
import inspect
import json
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_loader  # noqa: E402
from make_golden import encode_default  # noqa: E402

OUT_DIR = os.path.join(os.path.dirname(HERE), "tests", "golden")
SQRT2 = np.sqrt(2.0)


class _Scalar:
    def __init__(self, v):
        self.v = v

    def item(self):
        return self.v.item()


class _Coord:
    def __init__(self, v):
        self.data = self.values = np.asarray(v)

    def min(self):
        return _Scalar(self.data.min())

    def max(self):
        return _Scalar(self.data.max())


class _Surface:
    """What a_star_search reads of a DataArray: ndim, dims, shape, data, coords[name].data, raster[name], attrs."""

    def __init__(self, data, ys, xs, attrs):
        self.data = self.values = data
        self.shape = data.shape
        self.ndim = data.ndim
        self.dims = ("y", "x")
        self.coords = {"y": _Coord(ys), "x": _Coord(xs)}
        self.attrs = attrs

    def __getitem__(self, k):
        return self.coords[k]

    def __array__(self, dtype=None, copy=None):
        return self.data if dtype is None else self.data.astype(dtype)


def coords(h, w, ry, rx):
    return np.linspace((h - 1) * ry, 0, h), np.linspace(0, (w - 1) * rx, w)


def run(data, ry, rx, use_attrs, start, goal, barriers, conn, snap_start, snap_goal):
    """The reference's output and its warnings as (start warned, end warned)."""
    pf = ref_loader.load("pathfinding")
    ys, xs = coords(*data.shape, ry, rx)
    s = _Surface(data, ys, xs, {"res": (rx, ry)} if use_attrs else {})
    with warnings.catch_warnings(record=True) as ws:
        warnings.simplefilter("always")
        out = pf.a_star_search(s, start, goal, barriers, "x", "y", conn, snap_start, snap_goal)
    msgs = [str(w.message) for w in ws]
    return np.asarray(out.data), ("Start at a non crossable location" in msgs, "End at a non crossable location" in msgs)


def crossable(data, barriers):
    v = data.astype(np.float64)
    ok = ~np.isnan(v)
    for b in np.asarray(barriers, dtype=np.float64).ravel():
        ok &= v != b
    return ok


def moves(conn):
    if conn == 8:
        return [(-1, -1), (0, -1), (1, -1), (-1, 0), (1, 0), (-1, 1), (0, 1), (1, 1)]
    return [(0, -1), (-1, 0), (1, 0), (0, 1)]


def path_steps(out):
    """(a, b) of the path in an output: its cells ordered by value, each step orthogonal or diagonal."""
    idx = np.flatnonzero(~np.isnan(out.ravel()))
    if idx.size == 0:
        return -1, -1
    idx = idx[np.argsort(out.ravel()[idx], kind="stable")]
    r, c = np.divmod(idx, out.shape[1])
    diag = (np.diff(r) != 0) & (np.diff(c) != 0)
    return int((~diag).sum()), int(diag.sum())


def count_shortest(ok, conn, start, goal):
    """Number of shortest paths start -> goal (capped at 2), by an exact Dijkstra over (a, b) pairs: the float key
    orders the heap (pairs of lengths below 2^20 differ by far more than its rounding), equality is on pairs."""
    h, w = ok.shape
    dist = {start: (0, 0)}
    cnt = {start: 1}
    heap = [(0.0, start)]
    done = set()
    while heap:
        _, u = heapq.heappop(heap)
        if u in done:
            continue
        done.add(u)
        if u == goal:
            return cnt[u]
        a, b = dist[u]
        for dy, dx in moves(conn):
            v = (u[0] + dy, u[1] + dx)
            if not (0 <= v[0] < h and 0 <= v[1] < w) or not ok[v] or v in done:
                continue
            nd = (a, b + 1) if dy and dx else (a + 1, b)
            if v not in dist or nd[0] + nd[1] * SQRT2 < dist[v][0] + dist[v][1] * SQRT2 - 1e-9:
                dist[v], cnt[v] = nd, cnt[u]
                heapq.heappush(heap, (nd[0] + nd[1] * SQRT2, v))
            elif nd == dist[v]:
                cnt[v] = min(2, cnt[v] + cnt[u])
    return 0


class Cases:
    def __init__(self):
        self.cols = {k: [] for k in ("data", "barriers", "out")}
        self.off = {k: [0] for k in ("data", "barriers")}
        self.rows = []

    def add(self, data, ry, rx, use_attrs, sp, gp, barriers, conn, snap_start, snap_goal, start_cell, goal_cell):
        """One call; sp / gp are the (y, x) points, start_cell / goal_cell the cells they map to (before snapping)."""
        out, (ws, we) = run(data, ry, rx, use_attrs, sp, gp, barriers, conn, snap_start, snap_goal)
        a, b = path_steps(out)
        uniq = 0
        if a >= 0:
            idx = np.flatnonzero(~np.isnan(out.ravel()))
            first = idx[np.argmin(out.ravel()[idx])]
            last = idx[np.argmax(out.ravel()[idx])]
            s, g = divmod(int(first), data.shape[1]), divmod(int(last), data.shape[1])
            uniq = int(count_shortest(crossable(data, barriers), conn, s, g) == 1)
        bars = np.asarray(barriers, dtype=np.float64).ravel()
        self.cols["data"].append(data.astype(np.float64).ravel())
        self.cols["barriers"].append(bars)
        self.cols["out"].append(out.ravel())
        self.off["data"].append(self.off["data"][-1] + data.size)
        self.off["barriers"].append(self.off["barriers"][-1] + bars.size)
        self.rows.append((data.shape[0], data.shape[1], int(data.dtype.kind == "i"), conn, int(snap_start),
                          int(snap_goal), int(use_attrs), int(ws), int(we), a, b, uniq))
        self.pts = getattr(self, "pts", []) + [(ry, rx, sp[0], sp[1], gp[0], gp[1])]
        return out

    def arrays(self, prefix):
        return {prefix + "data": np.concatenate(self.cols["data"]),
                prefix + "barriers": np.concatenate(self.cols["barriers"]),
                prefix + "out": np.concatenate(self.cols["out"]),
                prefix + "data_off": np.array(self.off["data"], np.int64),
                prefix + "bar_off": np.array(self.off["barriers"], np.int64),
                # h, w, int cells, connectivity, snap_start, snap_goal, attrs, start warned, end warned, a, b, unique
                prefix + "meta": np.array(self.rows, np.int64),
                # ry, rx, start y, start x, goal y, goal x
                prefix + "pts": np.array(self.pts, np.float64)}


def point(h, w, ry, rx, cell, frac=0.0):
    ys, xs = coords(h, w, ry, rx)
    return (float(ys[cell[0]] - frac * ry), float(xs[cell[1]] + frac * rx))


DOC = np.array([[0, 1, 0, 0], [1, 1, 0, 0], [0, 1, 2, 2], [1, 0, 2, 0], [0, 2, 2, 2]])
NANS = np.array([[0, 1, 0, 0], [1, 1, np.nan, 0], [0, 1, 2, 2], [1, 0, 2, 0], [0, np.nan, 2, 2]])


def fixtures(cs):
    # the docstring: lat from 4 down to 0, lon 0..3, barriers [0], start (3, 0), goal (0, 1)
    cs.add(DOC, 1.0, 1.0, False, (3, 0), (0, 1), [0], 8, False, False, None, None)
    # test_a_star_search_connectivity and _snap: create_test_raster's res (0.5, 0.5), start (1.5, 1), goal (0, 0.5)
    for conn in (8, 4):
        for ss, sg in ((True, True), (False, False), (True, False), (False, True)):
            cs.add(NANS, 0.5, 0.5, True, (1.5, 1), (0, 0.5), [], conn, ss, sg, None, None)
    # test_a_star_search_with_barriers: start (2, 0), barriers [1], every goal
    ys, xs = coords(5, 4, 0.5, 0.5)
    for x1 in xs:
        for y1 in ys:
            if (y1, x1) != (2, 0):
                cs.add(DOC, 0.5, 0.5, True, (2, 0), (y1, x1), [1], 8, False, False, None, None)
    # test_a_star_search_no_barriers: every start and goal
    for x0 in xs:
        for y0 in ys:
            for x1 in xs:
                for y1 in ys:
                    cs.add(DOC, 0.5, 0.5, True, (y0, x0), (y1, x1), [], 8, False, False, None, None)


def small(cs, n=400):
    rng = np.random.default_rng(20261017)
    for k in range(n):
        h, w = (int(v) for v in rng.integers(2, 41 if k % 4 == 0 else 21, 2))
        conn = (4, 8)[k % 2]
        dens = float(rng.uniform(0.0, 0.45))
        fam = k % 5
        if fam == 0:     # integer cells, barrier value 1
            data = np.where(rng.random((h, w)) < dens, 1, rng.integers(2, 5, (h, w))).astype(np.int64)
            bars = [1]
        elif fam == 1:   # float cells with NaN obstacles, no barriers
            data = rng.normal(0, 1, (h, w))
            data[rng.random((h, w)) < dens] = np.nan
            bars = []
        elif fam == 2:   # float cells, float barriers, some NaN
            data = rng.choice([0.5, 1.0, 2.5, 3.0], (h, w), p=[0.3, 0.3, 0.2, 0.2]).astype(np.float64)
            data[rng.random((h, w)) < dens / 2] = np.nan
            bars = [2.5, 0.5] if dens > 0.2 else [2.5]
        elif fam == 3:   # integer cells, a barrier no cell has
            data = rng.integers(0, 3, (h, w)).astype(np.int64)
            bars = [7]
        else:            # integer cells, several int barriers
            data = rng.integers(0, 6, (h, w)).astype(np.int64)
            bars = [0, 5] if dens > 0.15 else [5]
        ry, rx = [(1.0, 1.0), (0.5, 0.5), (2.0, 0.25)][k % 3]
        use_attrs = k % 7 != 3 or h == 1 or w == 1
        s = (int(rng.integers(h)), int(rng.integers(w)))
        g = s if k % 23 == 0 else (int(rng.integers(h)), int(rng.integers(w)))
        if k % 6 == 0:
            s, g = (0, 0), (h - 1, w - 1)
        snap_s, snap_g = bool(k % 3 == 0), bool(k % 4 == 1)
        frac = 0.3 if k % 5 == 2 else 0.0
        cs.add(data, ry, rx, use_attrs, point(h, w, ry, rx, s, frac), point(h, w, ry, rx, g, frac), bars, conn,
               snap_s, snap_g, s, g)
    # only the opposite corner crossable: the snap finds nothing below the diagonal (NONE)
    for h, w in ((2, 2), (3, 5), (6, 4)):
        data = np.ones((h, w), np.int64)
        data[h - 1, w - 1] = 0
        for conn in (8, 4):
            cs.add(data, 1.0, 1.0, True, point(h, w, 1.0, 1.0, (0, 0)), point(h, w, 1.0, 1.0, (h - 1, w - 1)),
                   [1], conn, True, False, None, None)
            cs.add(data, 1.0, 1.0, True, point(h, w, 1.0, 1.0, (h - 1, w - 1)), point(h, w, 1.0, 1.0, (0, 0)),
                   [1], conn, False, True, None, None)


def large_raster(kind, h, w):
    """0/1 cells (barrier 1) for 'random' and 'maze'; int16 elevations with NaN water for 'dem'."""
    if kind == "random":
        rng = np.random.default_rng(99)
        data = (rng.random((h, w)) < 0.3).astype(np.int64)
        data[0, 0] = data[h - 1, w - 1] = 0
        return data
    if kind == "maze":   # serpentine: walls every 4th row, with a gap at alternating ends
        data = np.zeros((h, w), np.int64)
        for i, r in enumerate(range(2, h - 1, 4)):
            data[r, :] = 1
            data[r, (w - 2, w - 1) if i % 2 == 0 else (0, 1)] = 0
        return data
    i = np.arange(h)[:, None]
    j = np.arange(w)[None, :]
    z = (200 + 60 * np.sin(i / 23.0) * np.cos(j / 31.0) + 0.5 * ((i * 7 + j * 13) % 17)).astype(np.int16)
    z = z.astype(np.float64)
    z[(z < 170) & ((i + j) % 5 != 0)] = np.nan
    z[0, 0] = z[h - 1, w - 1] = 200.0
    return z


LARGE = [("random", 400, 400, 8), ("maze", 301, 240, 8), ("dem", 256, 256, 4)]


def large(g):
    for kind, h, w, conn in LARGE:
        data = large_raster(kind, h, w)
        bars = [1] if kind != "dem" else []
        cs = Cases()
        out = cs.add(data, 1.0, 1.0, True, point(h, w, 1.0, 1.0, (0, 0)), point(h, w, 1.0, 1.0, (h - 1, w - 1)),
                     bars, conn, False, False, None, None)
        idx = np.flatnonzero(~np.isnan(out.ravel()))
        g["large_%s_meta" % kind] = np.array(cs.rows[0], np.int64)
        g["large_%s_idx" % kind] = idx.astype(np.int32)
        g["large_%s_val" % kind] = out.ravel()[idx]
        if kind == "dem":
            g["large_dem_z"] = np.nan_to_num(data, nan=-1).astype(np.int16)
        else:
            g["large_%s_bits" % kind] = np.packbits(data.ravel().astype(bool))


def signature():
    pf = ref_loader.load("pathfinding")
    return {"a_star_search": [[k, encode_default(v.default)]
                              for k, v in inspect.signature(inspect.unwrap(pf.a_star_search)).parameters.items()]}


def main():
    cs = Cases()
    fixtures(cs)
    g = cs.arrays("fix_")
    cs = Cases()
    small(cs)
    g.update(cs.arrays("small_"))
    large(g)
    np.savez_compressed(os.path.join(OUT_DIR, "pathfinding_reference.npz"), **g)
    with open(os.path.join(OUT_DIR, "pathfinding_signature.json"), "w") as f:
        json.dump(signature(), f, indent=1, sort_keys=True)
        f.write("\n")
    m = g["small_meta"]
    print(len(m), "small cases:", int((m[:, 9] >= 0).sum()), "with a path,", int(m[:, 11].sum()), "unique")


if __name__ == "__main__":
    main()

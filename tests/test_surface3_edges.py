"""The 3x3 surface operators at nodata fills, extreme magnitudes and compass edges, against the CPU oracle.

slope (square and rectangular cells), aspect, curvature, hillshade, the fused suite, focal.mean (float32, float64,
float32 -> float64) and the 3x3 convolve run on rasters of terrain around 500 with fill values planted as single
cells, 1-cell-wide rows and columns, and blocks, at the raster edges, at the 128-cell strip edges, at the
2048-cell tile edge and at the row-segment edges.  Fill values are those real rasters use: NaN, -9999, the int16
and uint16 extremes, +-FLT_MAX (the float32 nodata of many GeoTIFFs) and +-DBL_MAX (inf once cast to float32).
The reference computes through them, so the kernels must too.

Each case runs on every path that serves it: the TMA kernel (aligned rows), the cp.async kernel (a base one cell
past alignment), the direct-ingest kernels reading int16 / uint16 / int32 / float64 cells, and the public API with
numpy (host-stencil runner) and torch inputs.  The C entry points read their input from inside a larger buffer of
large finite cells and write into sentinel buffers, so a read or write outside the raster shows up.

The oracle (oracle/oracle.py) restates the reference's float32 / float64 type rules; the CPU tests at the top
check it against a NumPy transcription of the reference formulas at every fill class first."""
import ctypes

import numpy as np
import pytest

import oracle as o
from helpers import (K_INGEST, K_STRIP_CPASYNC, K_STRIP_TMA, Pitched, assert_aspect_close, assert_close_f32,
                     gpu_lib, in_buffer, last_kind, raster, stream)

torch = pytest.importorskip("torch")

F32MAX = float(np.finfo(np.float32).max)   # 3.4028235e38
F64MAX = float(np.finfo(np.float64).max)   # 1.7976931348623157e308: astype(float32) makes it inf
CELLS = (10.0, 25.5)
SUNS = [(225, 25), (315, 45), (0, 25), (90, 25), (180, 25), (270, 25), (360, 25), (225, 1), (225, 90)]
TYPED = {np.dtype(np.int16): 4, np.dtype(np.uint16): 5, np.dtype(np.int32): 2, np.dtype(np.float64): 1}

# fill value -> the cell type it lives in
FILLS = {
    "nan": (np.float32, np.nan),
    "-9999": (np.float32, -9999.0),
    "int16 min": (np.int16, -32768),
    "int16 max": (np.int16, 32767),
    "uint16 0": (np.uint16, 0),
    "uint16 max": (np.uint16, 65535),
    "+FLT_MAX": (np.float32, F32MAX),
    "-FLT_MAX": (np.float32, -F32MAX),
    "+DBL_MAX": (np.float64, F64MAX),
    "-DBL_MAX": (np.float64, -F64MAX),
}


# ----------------------------------------------------------------------------------- reference transcription
def _ring(core, dtype, fill=np.nan):
    out = np.full((core.shape[0] + 2, core.shape[1] + 2), fill, dtype)
    out[1:-1, 1:-1] = core
    return out


def ref_x(d, a_row_below):
    """The reference's X = 8 dz_dx, (c + 2 f + i) - (a + 2 d + g), summed column by column in float64; a, b, c
    are row y+1 in slope (a_row_below) and row y-1 in aspect."""
    top, bot = (d[2:], d[:-2]) if a_row_below else (d[:-2], d[2:])
    return (top[:, 2:] + 2 * d[1:-1, 2:] + bot[:, 2:]) - (top[:, :-2] + 2 * d[1:-1, :-2] + bot[:, :-2])


def rows_x(d):
    """X as the kernels form it: exact per-row differences D = r - l, then (2 D(y) + D(y-1)) + D(y+1)."""
    D = d[:, 2:] - d[:, :-2]
    return (2 * D[1:-1] + D[:-2]) + D[2:]


def ref_slope(data, csx, csy, x=None):
    """slope.py `_cpu`: a, b, c = row y+1; Numba promotes `2 * f32` to float64.  `x` replaces the numerator
    of dz_dx."""
    d = data.astype(np.float32).astype(np.float64)
    a, b, c = d[2:, :-2], d[2:, 1:-1], d[2:, 2:]
    g, h, i = d[:-2, :-2], d[:-2, 1:-1], d[:-2, 2:]
    dz_dx = (ref_x(d, True) if x is None else x) / (8 * csx)
    dz_dy = ((g + 2 * h + i) - (a + 2 * b + c)) / (8 * csy)
    p = (dz_dx * dz_dx + dz_dy * dz_dy) ** .5
    return _ring((np.arctan(p) * 57.29578).astype(np.float32), np.float32)


def ref_aspect(data, x=None):
    """aspect.py `_run_numpy`: a, b, c = row y-1; flat -> -1; compass fold of atan2(dz_dy, -dz_dx)."""
    d = data.astype(np.float32).astype(np.float64)
    a, b, c = d[:-2, :-2], d[:-2, 1:-1], d[:-2, 2:]
    g, h, i = d[2:, :-2], d[2:, 1:-1], d[2:, 2:]
    dz_dx = (ref_x(d, False) if x is None else x) / 8
    dz_dy = ((g + 2 * h + i) - (a + 2 * b + c)) / 8
    asp = np.arctan2(dz_dy, -dz_dx) * (180.0 / np.pi)
    comp = np.where(asp < 0, 90.0 - asp, np.where(asp > 90.0, 360.0 - asp + 90.0, 90.0 - asp))
    comp = np.where((dz_dx == 0) & (dz_dy == 0), -1.0, comp)
    return _ring(comp.astype(np.float32), np.float32)


def ref_curvature(data, cellsize):
    """curvature.py `_cpu`: the neighbour sums are float32; `/ 2` promotes to float64."""
    d = data.astype(np.float32)
    ctr = d[1:-1, 1:-1].astype(np.float64)
    ns = (d[2:, 1:-1] + d[:-2, 1:-1]).astype(np.float64)
    ew = (d[1:-1, 2:] + d[1:-1, :-2]).astype(np.float64)
    dd = ns / 2 - ctr
    e = ew / 2 - ctr
    return _ring((-2 * (dd + e) * 100 / (cellsize * cellsize)).astype(np.float32), np.float32)


def ref_hillshade(data, azimuth=225, angle_altitude=25):
    """hillshade.py `_run_numpy`, as written there."""
    data = data.astype(np.float32)
    azimuth = 360.0 - azimuth
    x, y = np.gradient(data)
    slope = np.pi / 2. - np.arctan(np.sqrt(x * x + y * y))
    aspect = np.arctan2(-x, y)
    azimuthrad = azimuth * np.pi / 180.
    altituderad = angle_altitude * np.pi / 180.
    shaded = np.sin(altituderad) * np.sin(slope) + \
        np.cos(altituderad) * np.cos(slope) * np.cos((azimuthrad - np.pi / 2.) - aspect)
    result = (shaded + 1) / 2
    result[(0, -1), :] = np.nan
    result[:, (0, -1)] = np.nan
    return result


def ref_focal_mean(data, excludes):
    """focal.py `_mean_numpy` on `data.astype(float)`: excluded centres copied, else the sequential nanmean of
    the window clamped to the raster."""
    d = data.astype(np.float64)
    H, W = d.shape
    out = np.empty_like(d)
    for y in range(H):
        for x in range(W):
            v = d[y, x]
            if any(v == e or (np.isnan(v) and np.isnan(e)) for e in excludes):
                out[y, x] = v
                continue
            s, n = 0.0, 0
            for u in d[max(y - 1, 0):y + 2, max(x - 1, 0):x + 2].ravel():
                if not np.isnan(u):
                    s += u
                    n += 1
            out[y, x] = s / n if n else np.nan
    return out


# ----------------------------------------------------------------------------------------------- inputs
def _terrain(H, W, seed, dtype=np.float32):
    z = raster(H, W, seed, nan_frac=0.0)
    if np.dtype(dtype).kind in "iu":
        z = np.round(z).clip(np.iinfo(dtype).min + 1, np.iinfo(dtype).max - 1)
    return z.astype(dtype)


def _layouts(H, W, segs):
    """Where fills are planted: {layout: [(row slice, col slice), ...]}.  Edges of the raster, of the 128-cell
    strips (127 / 128), of the 2048-cell tile (2047 / 2048) when W reaches it, and the first rows of the row
    segments `segs`."""
    cols = [0, 1, 127, 128, W - 2, W - 1] + ([2047, 2048] if W > 2049 else [])
    rows = sorted({0, 1, H // 2 + 3, H - 2, H - 1} | {r for s in segs for r in (s - 1, s)})
    mid_c = W // 2 + 37
    cells = [(slice(r, r + 1), slice(c, c + 1)) for r in rows for c in cols if 0 <= r < H and 0 <= c < W]
    cells.append((slice(H // 2 - 5, H // 2 - 4), slice(mid_c, mid_c + 1)))   # an isolated cell
    lines_r = [(slice(r, r + 1), slice(None)) for r in sorted({0, H // 2 - 9, H - 1} | set(segs)) if r < H]
    lines_c = [(slice(None), slice(c, c + 1)) for c in [0, 127, W - 1] + ([2048] if W > 2049 else [])]
    blocks = [(slice(0, 4), slice(0, 5)), (slice(H - 4, H), slice(W - 5, W)),
              (slice(H // 2, H // 2 + 7), slice(60, 64))]
    blocks += [(slice(max(s - 2, 0), s + 3), slice(125, 131)) for s in segs]
    if W > 2049:
        blocks.append((slice(1, 6), slice(2045, 2051)))
    return {"cells": cells, "rows": lines_r, "cols": lines_c, "blocks": blocks}


def planted(dtype, value, H, W, seed, segs):
    """{layout: raster of `dtype` cells with `value` planted}."""
    out = {}
    for name, spots in _layouts(H, W, segs).items():
        z = _terrain(H, W, seed, dtype)
        for r, c in spots:
            z[r, c] = value
        out[name] = z
    return out


def magnitude_rasters(H, W, seed):
    """Terrain offset by 1e6 and 1.6e7 (float32 ulp 0.06 and 2: X and Y cancel), and int32 cells near +-2^31
    and 2^24 (where int -> float32 rounds)."""
    base = raster(H, W, seed, nan_frac=0.0).astype(np.float64) - 500.0
    big = np.round(base * 40.0)
    return {
        "offset 1e6": (base + 1e6).astype(np.float32),
        "offset 1.6e7": (base + 1.6e7).astype(np.float32),
        "int32 near 2^31": (2 ** 31 - 1 - np.abs(big) * 3).astype(np.int32),
        "int32 near -2^31": (-2 ** 31 + np.abs(big) * 3).astype(np.int32),
        "int32 near 2^24": (2 ** 24 + np.round(base)).astype(np.int32),
    }


def compass_rasters(H, W):
    """Planes whose gradient points along each of 16 directions, exactly along the diagonals (|X| == |Y|) and
    along the axes; -0.0 cells in a flat zero field; a flat field next to NaN cells."""
    yy, xx = np.mgrid[:H, :W].astype(np.float64)
    out = {}
    for k in range(16):
        t = np.deg2rad(22.5 * k)
        gx, gy = np.round(40 * np.cos(t)), np.round(40 * np.sin(t))
        if k % 4 == 2:
            gy = np.copysign(abs(gx), gy)        # exactly diagonal
        out["plane %g deg" % (22.5 * k)] = (500 + gx * xx + gy * yy).astype(np.float32)
    zero = np.zeros((H, W), np.float32)
    zero[::3, ::2] = np.float32(-0.0)
    zero[5:9, 100:140] = np.float32(-0.0)
    out["signed zeros"] = zero
    flat = np.full((H, W), 500.0, np.float32)
    flat[::7, ::11] = np.nan
    flat[H // 2, :] = np.nan
    out["flat next to NaN"] = flat
    return out


# ------------------------------------------------------------------------------ oracle vs transcription (CPU)
@pytest.mark.parametrize("fill", list(FILLS))
def test_oracle_matches_reference_formulas_at_fills(fill):
    """The oracle gives the reference's values at each fill class: slope, aspect, curvature and hillshade within
    the parity bars of the GPU tests, focal.mean bit for bit."""
    dtype, value = FILLS[fill]
    H, W = 14, 132
    for layout, src in planted(dtype, value, H, W, 3, [6]).items():
        with np.errstate(all="ignore"):
            z = src.astype(np.float32)
            what = "%s %s" % (fill, layout)
            assert_close_f32(o.slope(z, *CELLS), ref_slope(src, *CELLS), what="slope " + what)
            assert_aspect_close(o.aspect(z), ref_aspect(src), what="aspect " + what)
            assert_close_f32(o.curvature(z, 10.0), ref_curvature(src, 10.0), what="curvature " + what)
            for az, alt in ((225, 25), (90, 1)):
                assert_close_f32(o.hillshade(z, az, alt), ref_hillshade(src, az, alt), what="hillshade " + what)
            for ex in ((np.nan,), (np.nan, -9999.0)):
                np.testing.assert_array_equal(o.focal_mean(src, excludes=ex), ref_focal_mean(src, ex),
                                              err_msg="focal.mean " + what)


def test_oracle_matches_reference_formulas_at_magnitudes_and_compass_edges():
    H, W = 12, 132
    cases = dict(magnitude_rasters(H, W, 5))
    cases.update(compass_rasters(H, W))
    for name, src in cases.items():
        z = src.astype(np.float32)
        with np.errstate(all="ignore"):
            assert_close_f32(o.slope(z, *CELLS), ref_slope(src, *CELLS), what="slope " + name)
            assert_aspect_close(o.aspect(z), ref_aspect(src), what="aspect " + name)
            assert_close_f32(o.curvature(z, 10.0), ref_curvature(src, 10.0), what="curvature " + name)
            assert_close_f32(o.hillshade(z), ref_hillshade(src), what="hillshade " + name)
            np.testing.assert_array_equal(o.focal_mean(src), ref_focal_mean(src, (np.nan,)), err_msg=name)


def test_transcription_sees_the_fill_value_effects():
    """The transcription itself is not vacuous at FLT_MAX: hillshade's float32 x*x + y*y overflows there (slope
    0, value (cos(alt) cos(A - aspect) + 1) / 2, not 0.5), and a cell diagonal to the fill has |X| == |Y| far
    beyond 2^126 and an aspect on the diagonal."""
    z = np.full((5, 5), 500.0, np.float32)
    z[2, 2] = -F32MAX
    with np.errstate(all="ignore"):
        hs = ref_hillshade(z)
        asp = ref_aspect(z)
    assert abs(hs[1, 2] - 0.5) > 0.2 and abs(hs[2, 1] - 0.5) > 0.2
    assert np.isclose(hs[1, 2] + hs[3, 2], 1.0) and np.isclose(hs[2, 1] + hs[2, 3], 1.0)
    np.testing.assert_allclose([asp[1, 1], asp[1, 3], asp[3, 1], asp[3, 3]], [135, 225, 45, 315], atol=1e-4)
    # a row of the fill through terrain: the reference's column sums lose the terrain, the row differences not
    z = np.full((3, 5), 500.0, np.float32) + np.arange(5, dtype=np.float32)
    z[1] = -F32MAX
    d = z.astype(np.float64)
    np.testing.assert_array_equal(ref_x(d, True), 0.0)
    np.testing.assert_array_equal(rows_x(d), 4.0)


# ---------------------------------------------------------------------------------------------- GPU harness
@pytest.fixture(scope="module")
def lib():
    return gpu_lib()


def _seg_starts(lib, H, W):
    """First rows of the row segments of every kernel these tests run (surface.cu `geometry`, stencil3.cuh):
    TMA (tile width, rows per stage, CTAs per SM) for the float32 operators, the suite, float64 output and the
    direct-ingest kernels, and the cp.async kernel's segments for 4- and 8-byte cells."""
    n = ctypes.c_int(0)
    lib.check(lib.lib().xrs_device_sm_count(0, ctypes.byref(n)))
    sm = n.value
    heights = set()
    for tile, rows, ctas in ((2048, 4, 1), (1536, 8, 1), (2048, 2, 1), (1024, 4, 2), (1024, 2, 2)):
        heights.add(int(lib.lib().xrs_debug_pick_seg_rows(H, (W + tile - 1) // tile, sm * ctas, 32, 2, rows, 2)))
    strips = (W + 127) // 128
    for fr in (4, 2):                         # cp.async: kFallbackRows, or 2 rows of 8-byte cells
        want = (sm * 2 * 8 * 8 + strips - 1) // strips
        h = min(max((H + want - 1) // want, 64), H)
        heights.add(max((h + 2 + fr - 1) // fr * fr - 2, 1))
    return sorted({k * h for h in heights for k in range(1, H // h + 1) if k * h < H})


def _launch(lib, fn, H, W, kind, what, itemsize=4):
    """fn(out_ptr, out_pitch) into a sentinel buffer; checks the kernel that ran and the untouched border."""
    out = Pitched(H, W, itemsize)
    fn(out.ptr, out.pitch)
    torch.cuda.synchronize()
    got = last_kind(lib)
    assert got == kind, "%s: kernel %d ran, expected %d" % (what, got, kind)
    return out.inside(what).view(np.float32 if itemsize == 4 else np.float64)


class Case(object):
    """One raster on the device in the layouts each path needs: float32 aligned (TMA) and shifted by one cell
    (cp.async), and its source cells for direct ingest (int16 / uint16 / int32 as they are, float64 for float
    sources)."""

    def __init__(self, src):
        self.src = src
        self.z = src.astype(np.float32)
        self.H, self.W = src.shape
        # every input has a guard row above and below and guard cells right of each row (16-byte pitch)
        self.tma = in_buffer(self.z, pad_cols=4, rows_above=1, rows_below=1)
        self.cpa = in_buffer(self.z, pad_cols=3, rows_above=1, rows_below=1, shift=1)
        ing = src if src.dtype in TYPED else src.astype(np.float64)
        pad = (-(self.W * ing.itemsize) % 16) // ing.itemsize or 16 // ing.itemsize
        t, ptr, pitch = in_buffer(ing, pad_cols=pad, rows_above=1, rows_below=1)
        self.ing = (t, ptr, TYPED[ing.dtype], pitch)
        self.f64 = in_buffer(src.astype(np.float64), pad_cols=2, rows_above=1, rows_below=1)
        self.f64_cpa = in_buffer(src.astype(np.float64), pad_cols=1, rows_above=1, rows_below=1, shift=1)

    def paths(self, lib, call, what, itemsize=4, f64_in=False):
        """call(in_ptr, in_pitch, out_ptr, out_pitch) on the TMA and the cp.async kernel."""
        a, b = (self.f64, self.f64_cpa) if f64_in else (self.tma, self.cpa)
        H, W = self.H, self.W
        return [(what + " tma", _launch(lib, lambda op, p: call(a[1], a[2], op, p), H, W, K_STRIP_TMA, what,
                                        itemsize)),
                (what + " cp.async", _launch(lib, lambda op, p: call(b[1], b[2], op, p), H, W, K_STRIP_CPASYNC,
                                             what, itemsize))]

    def ingest(self, lib, op, par, what):
        t, ptr, code, pitch = self.ing
        p = np.asarray(par, dtype=np.float64)
        return (what + " ingest %s" % t.dtype,
                _launch(lib, lambda o_, op_: lib.call("xrs_surface_typed", op, ptr, code, pitch, o_, op_,
                                                      self.H, self.W, p.ctypes.data, stream()),
                        self.H, self.W, K_INGEST, what))


def _api(src, fn):
    """The public function on the raster as a numpy array (host-stencil runner) and as a device tensor."""
    import xrspatial_b200 as xb
    res = []
    for kind, data in (("numpy", src), ("torch", torch.from_numpy(np.ascontiguousarray(src)).cuda())):
        agg = xb.DataArray(data, dims=("y", "x"), attrs={"res": (10.0, 10.0)})
        r = fn(xb, agg).data
        res.append(("api " + kind, np.asarray(r.cpu().numpy() if hasattr(r, "cpu") else r)))
    return res


def _mean_bound(got, ref, src, what):
    """float64 focal.mean: the kernel adds row sums where the reference adds in sequence.  Each cell passes
    through at most 4 roundings in the kernel's tree and 8 in the reference's sequence, so the two quotients
    differ by at most (4 + 8) 2^-53 sum|x| / n plus the final rounding; non-finite results and excluded cells
    match exactly.  The tighter 3 2^-53 sum|x| / n does not hold: in test_focal_mean_f64_cancelling_window a
    window of 1e16, 1 and -1e16 cells differs by 1.0 in the two orders where it would allow 0.74."""
    d = src.astype(np.float64)
    ok = ~np.isnan(d)
    a = np.pad(np.where(ok, np.abs(d), 0.0), 1)
    c = np.pad(ok.astype(np.float64), 1)
    H, W = d.shape
    with np.errstate(all="ignore"):
        s = sum(a[i:i + H, j:j + W] for i in range(3) for j in range(3))
        n = sum(c[i:i + H, j:j + W] for i in range(3) for j in range(3))
        bound = 12 * 2.0 ** -53 * s / n + np.spacing(np.abs(ref))
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref), err_msg=what + ": NaN masks differ")
    fin = np.isfinite(ref)
    np.testing.assert_array_equal(got[~fin & ~np.isnan(ref)], ref[~fin & ~np.isnan(ref)], err_msg=what)
    err = np.abs(got[fin] - ref[fin])
    bad = ~(err <= bound[fin])
    assert not bad.any(), "%s: %d windows beyond the summation-order bound, first at %s: %r vs %r" % (
        what, int(bad.sum()), tuple(np.argwhere(fin)[np.argmax(bad)]), got[fin][bad][0], ref[fin][bad][0])


def _f32_bits(got, ref, what):
    """float32 focal.mean: the oracle rounded to float32, bit for bit (NaN payloads aside)."""
    r = ref.astype(np.float32)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(r), err_msg=what + ": NaN masks differ")
    m = ~np.isnan(r)
    bad = got[m].view(np.uint32) != r[m].view(np.uint32)
    assert not bad.any(), "%s: %d cells differ, first at %s: %r vs %r" % (
        what, int(bad.sum()), tuple(np.argwhere(m)[np.argmax(bad)]), got[m][bad][0], r[m][bad][0])


def _fail_cells(got, ref, what, aspect=False):
    """Run the gate; on failure name the first cells that broke it."""
    try:
        (assert_aspect_close if aspect else assert_close_f32)(got, ref, what=what)
    except AssertionError as e:
        g, r = np.asarray(got, np.float64), np.asarray(ref, np.float64)
        with np.errstate(all="ignore"):
            d = np.abs(g - r)
            if aspect:
                d = np.minimum(d, 360 - d)
            bad = ~((d <= 1e-5 * np.abs(r) + (1e-4 if aspect else 1e-6)) | (np.isnan(g) & np.isnan(r)) | (g == r))
        cells = ["%s: %r vs %r" % (tuple(int(v) for v in i), g[tuple(i)], r[tuple(i)]) for i in np.argwhere(bad)[:6]]
        raise AssertionError("%s\n  first cells (kernel vs oracle): %s" % (e, "; ".join(cells)))


def kernel_x(orc, z, op, *args):
    """The oracle's slope or aspect, except in windows where the reference's column-by-column float64 X and
    the kernels' row-by-row X differ (cells more than 2^29 apart in one window, e.g. a row of -FLT_MAX through
    terrain: the reference's sums round the terrain away).  There the kernels give the reference's formula
    on their own X, which is the exact Horn sum when the row differences are exact (DESIGN.md 4.1, fill
    values)."""
    d = z.astype(np.float64)
    with np.errstate(all="ignore"):
        xr, xf = rows_x(d), ref_x(d, op == "slope")
        differ = _ring(~((xr == xf) | (np.isnan(xr) & np.isnan(xf))), bool, False)
        if not differ.any():
            return orc
        alt = ref_slope(z, *args, x=xr) if op == "slope" else ref_aspect(z, x=xr)
    return np.where(differ, alt, orc)


def check_surface(lib, case, what, ingest=True, api=True):
    """Every 3x3 surface operator on every path against the oracle."""
    z, H, W = case.z, case.H, case.W
    with np.errstate(all="ignore"):
        slope_sq = kernel_x(o.slope(z, 10.0, 10.0), z, "slope", 10.0, 10.0)
        slope_rc = kernel_x(o.slope(z, *CELLS), z, "slope", *CELLS)
        asp, curv = kernel_x(o.aspect(z), z, "aspect"), o.curvature(z, 10.0)
        curv_suite = o.curvature(z, (CELLS[0] + CELLS[1]) / 2)
        hills = {sun: o.hillshade(z, *sun) for sun in SUNS}
    ops = [
        ("slope square", 0, (10.0, 10.0), slope_sq,
         lambda i, ip, op, p: lib.call("xrs_slope_f32", i, ip, op, p, H, W, 10.0, 10.0, stream())),
        ("slope rect", 0, CELLS, slope_rc,
         lambda i, ip, op, p: lib.call("xrs_slope_f32", i, ip, op, p, H, W, CELLS[0], CELLS[1], stream())),
        ("aspect", 1, (), asp, lambda i, ip, op, p: lib.call("xrs_aspect_f32", i, ip, op, p, H, W, stream())),
        ("curvature", 2, (10.0,), curv,
         lambda i, ip, op, p: lib.call("xrs_curvature_f32", i, ip, op, p, H, W, 10.0, stream())),
    ]
    for sun in SUNS:
        ops.append(("hillshade %s" % (sun,), 3, sun, hills[sun],
                    lambda i, ip, op, p, sun=sun: lib.call("xrs_hillshade_f32", i, ip, op, p, H, W, float(sun[0]),
                                                           float(sun[1]), stream())))
    for name, code, par, ref, call in ops:
        label = "%s %s" % (name, what)
        res = case.paths(lib, call, label)
        if ingest:
            res.append(case.ingest(lib, code, par if par else (0.0,), label))
        for path, got in res:
            _fail_cells(got, ref, path, aspect=(code == 1))

    # the fused suite: all four outputs, then each alone with the other three NULL
    refs = [slope_rc, asp, curv_suite, hills[(225, 25)]]
    for only in (None, 0, 1, 2, 3):
        label = "suite %s %s" % ("all" if only is None else ["slope", "aspect", "curvature", "hillshade"][only], what)
        a, b = case.tma, case.cpa
        for (ptr, pitch), kind, tag in (((a[1], a[2]), K_STRIP_TMA, "tma"), ((b[1], b[2]), K_STRIP_CPASYNC, "cp.async")):
            outs = [Pitched(H, W) for _ in range(4)]
            ptrs = [outs[k].ptr if only in (None, k) else None for k in range(4)]
            lib.call("xrs_surface_suite_f32", ptr, pitch, *ptrs, outs[0].pitch, H, W, CELLS[0], CELLS[1], 225.0, 25.0,
                     stream())
            torch.cuda.synchronize()
            assert last_kind(lib) == kind, label
            for k in range(4):
                got = outs[k].inside(label).view(np.float32)
                if only not in (None, k):
                    assert (got.view(np.uint8) == 0x5A).all(), "%s: output %d was NULL but written" % (label, k)
                    continue
                _fail_cells(got, refs[k], "%s %s output %d" % (label, tag, k), aspect=(k == 1))

    if api:
        for name, fn, ref, aspect in (
                ("slope", lambda xb, agg: xb.slope(agg), slope_sq, False),
                ("aspect", lambda xb, agg: xb.aspect(agg), asp, True),
                ("curvature", lambda xb, agg: xb.curvature(agg), curv, False),
                ("hillshade", lambda xb, agg: xb.hillshade(agg, 315, 45), hills[(315, 45)], False)):
            for path, got in _api(case.src, fn):
                _fail_cells(got, ref, "%s %s %s" % (name, what, path), aspect=aspect)


def check_mean_conv(lib, case, what, api=True):
    """focal.mean in float32, float64 and float32 -> float64, with excludes [nan] and [nan, -9999]; the 3x3
    convolve."""
    H, W = case.H, case.W
    src64 = case.src.astype(np.float64)
    for ex in ((np.nan,), (np.nan, -9999.0)):
        e = np.array(ex, dtype=np.float64)
        label = "focal.mean excludes=%s %s" % (list(ex), what)
        ref32 = o.focal_mean(case.z, excludes=ex)
        ref64 = o.focal_mean(src64, excludes=ex)
        for path, got in case.paths(lib, lambda i, ip, op, p: lib.call("xrs_focal_mean_f32", i, ip, op, p, H, W,
                                                                      e.ctypes.data, len(e), stream()), label):
            _f32_bits(got, ref32, path + " f32")
        for path, got in case.paths(lib, lambda i, ip, op, p: lib.call("xrs_focal_mean_f32_f64", i, ip, op, p, H, W,
                                                                      e.ctypes.data, len(e), stream()),
                                    label, itemsize=8):
            _mean_bound(got, ref32, case.z, path + " f32->f64")
        for path, got in case.paths(lib, lambda i, ip, op, p: lib.call("xrs_focal_mean_f64", i, ip, op, p, H, W,
                                                                      e.ctypes.data, len(e), stream()),
                                    label, itemsize=8, f64_in=True):
            _mean_bound(got, ref64, src64, path + " f64")
        if api:
            for path, got in _api(case.src, lambda xb, agg: xb.mean(agg, excludes=list(ex))):
                if got.dtype == np.float32:     # a device raster of float32 or of integers cast to float32
                    _f32_bits(got, ref32, "%s %s" % (label, path))
                else:                           # float64 out: the raster's own cells widened
                    _mean_bound(got, ref64, src64, "%s %s" % (label, path))
    k = np.array([[0.3, -0.7, 0.11], [1.25, -0.5, 0.2], [-0.13, 0.9, -0.05]])
    ref = o.convolve_2d_fma(case.z, k)
    for path, got in case.paths(lib, lambda i, ip, op, p: lib.call("xrs_convolve2d_f32", i, ip, op, p, H, W,
                                                                  k.ctypes.data, 3, 3, stream()), "conv3 " + what):
        np.testing.assert_array_equal(np.isnan(got), np.isnan(ref), err_msg=path)
        m = ~np.isnan(ref)
        np.testing.assert_array_equal(got[m].view(np.uint32), ref[m].view(np.uint32), err_msg=path)


# ----------------------------------------------------------------------------------------------- GPU tests
H0, W0 = 72, 260


@pytest.mark.gpu
@pytest.mark.parametrize("fill", list(FILLS))
def test_fill_values(lib, fill):
    dtype, value = FILLS[fill]
    for layout, src in planted(dtype, value, H0, W0, 11, _seg_starts(lib, H0, W0)).items():
        case = Case(src)
        check_surface(lib, case, "%s %s" % (fill, layout), api=(layout == "blocks"))
        check_mean_conv(lib, case, "%s %s" % (fill, layout), api=(layout == "blocks"))


@pytest.mark.gpu
@pytest.mark.parametrize("fill", ["nan", "-FLT_MAX", "+DBL_MAX", "uint16 max"])
def test_fill_values_at_the_tile_edge(lib, fill):
    """Columns 2047 / 2048, where one 16-warp CTA tile ends and the next begins."""
    dtype, value = FILLS[fill]
    H, W = 9, 4100
    for layout, src in planted(dtype, value, H, W, 17, _seg_starts(lib, H, W) or [4]).items():
        case = Case(src)
        check_surface(lib, case, "%s %s W %d" % (fill, layout, W), api=False)
        check_mean_conv(lib, case, "%s %s W %d" % (fill, layout, W), api=False)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(magnitude_rasters(4, 8, 0)))
def test_magnitudes(lib, name):
    case = Case(magnitude_rasters(H0, W0, 23)[name])
    check_surface(lib, case, name)
    check_mean_conv(lib, case, name)


@pytest.mark.gpu
def test_compass_edges(lib):
    for name, src in compass_rasters(H0, W0).items():
        case = Case(src)
        check_surface(lib, case, name, api=False)
        check_mean_conv(lib, case, name, api=False)


@pytest.mark.gpu
def test_focal_mean_f64_cancelling_window(lib):
    """1e16, 1 and -1e16 in one window: the row sums cancel in another order than the reference's sequence, so
    the float64 result is held to the summation-order bound rather than to a relative tolerance.  Windows of
    -0.0 cells and of infinite sums are covered by test_compass_edges and the DBL_MAX fills."""
    H, W = 12, 132
    z = _terrain(H, W, 29).astype(np.float64)
    z[4, 10:13] = [1e16, 1.0, -1e16]
    z[5, 10], z[6, 12] = 1e16, -1e16
    z[8, 127:130] = [-1e16, 3.0, 1e16]
    case = Case(z)
    e = np.array([np.nan])
    ref = o.focal_mean(z)
    for path, got in case.paths(lib, lambda i, ip, op, p: lib.call("xrs_focal_mean_f64", i, ip, op, p, H, W,
                                                                  e.ctypes.data, 1, stream()),
                                "focal.mean cancelling", itemsize=8, f64_in=True):
        _mean_bound(got, ref, z, path)

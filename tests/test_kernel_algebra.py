"""CPU checks of the algebra the CUDA kernels use where it differs in FORM from the reference's
(the GPU parity tests check the kernels themselves): NumPy statements of the kernel arithmetic
against the pinned oracle, and the polynomial constants parsed out of the CUDA header."""
import os
import re

import numpy as np
import pytest

import oracle as o
from helpers import box_magnitude_fields, box_plant, box_planted_values, box_window_errors, terrain

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "xarray-spatial_b200", "csrc")


def _atan_coeffs():
    src = open(os.path.join(CSRC, "common.cuh")).read()
    body = src[src.index("float atan_poly01(float z)"):]
    body = body[:body.index("return p;")]
    c = [float(x) for x in re.findall(r"(-?\d\.\d+e[+-]\d+)f \* k", body)]
    assert len(c) == 8, c
    return c                      # highest degree first


def test_atan_polynomial_of_the_header_is_accurate_in_float32():
    """atan(t)/t on [0, 1] as a degree-7 polynomial in t^2 (common.cuh): 2.5e-7 relative when
    evaluated with float32 FMAs-free Horner steps, far inside the 1e-5 parity bar."""
    c = np.array(_atan_coeffs(), dtype=np.float32)
    t = np.linspace(0.0, 1.0, 200001, dtype=np.float32)
    z = (t * t).astype(np.float32)
    p = np.full_like(z, c[0])
    for k in c[1:]:
        p = (p * z + k).astype(np.float32)
    got = (t * p).astype(np.float64)
    ref = np.arctan(t.astype(np.float64))
    rel = np.abs(got[1:] - ref[1:]) / ref[1:]
    assert rel.max() < 4e-7, rel.max()


def _fma32(a, b, c):
    return np.float32(np.float64(a) * np.float64(b) + np.float64(c))   # one rounding, like FFMA


def _compass(u, v, coeffs):
    """NumPy statement of compass_deg (common.cuh): octant reduction, sign folded into t, polynomial
    and one fused multiply-add for the tail, float32.  The flat test is NaN-safe."""
    u, v = np.float32(u), np.float32(v)
    au, av = abs(u), abs(v)
    swap = au > av
    mx, mn = (au, av) if swap else (av, au)
    with np.errstate(divide="ignore", invalid="ignore"):
        t = np.float32(mn / mx)
    sgn = bool(np.signbit(u)) != bool(np.signbit(v))
    sgn = (not sgn) if swap else sgn
    ts = -t if sgn else t
    z = np.float32(ts * ts)
    p = np.float32(coeffs[0] * np.float32(57.29578))
    for k in coeffs[1:]:
        p = _fma32(p, z, np.float32(k * np.float32(57.29578)))
    if swap:
        k0 = 90.0 if u > 0 else 270.0
    else:
        k0 = (360.0 if u < 0 else 0.0) if v > 0 else 180.0
    r = _fma32(ts, p, np.float32(k0))
    return np.float32(-1.0) if (au == 0 and av == 0) else r


def test_compass_of_a_nan_sum_is_nan_not_flat():
    """aspect.py:74-88: `dz_dx == 0 and dz_dy == 0` is false when one Horn sum is NaN, and
    atan2(0, NaN) is NaN -- an isolated nodata pixel on a plateau must not read as flat (-1)."""
    coeffs = [np.float32(x) for x in _atan_coeffs()]
    for u, v in ((np.nan, 0.0), (0.0, np.nan), (np.nan, np.nan), (np.nan, 3.0), (-2.0, np.nan)):
        assert np.isnan(_compass(u, v, coeffs)), (u, v)
    z = np.full((5, 7), 100.0, dtype=np.float32)
    z[2, 3] = np.nan
    ref = o.aspect(z)
    assert np.isnan(ref[2, 2]) and np.isnan(ref[2, 4]) and np.isnan(ref[1, 3])   # W / E / N neighbours of the hole
    assert ref[1, 1] == -1.0 if not np.isnan(ref[1, 1]) else True


def test_compass_fold_matches_the_reference_branches():
    """aspect.py:74-88 maps atan2(dz_dy, -dz_dx) through three branches; the kernel evaluates
    atan2(-X, Y) folded to [0, 360) per octant.  Same angles on a dense fan of directions, including
    the axes and exact zeros."""
    coeffs = [np.float32(x) for x in _atan_coeffs()]
    rng = np.random.default_rng(0)
    pts = [(x, y) for x in (-3.0, -1.0, -1e-20, 0.0, 1e-20, 1.0, 2.5) for y in (-2.0, -1.0, 0.0, 1e-20, 1.0, 7.0)]
    pts += list(zip(rng.standard_normal(2000) * 10.0 ** rng.integers(-6, 6, 2000), rng.standard_normal(2000)))
    for X, Y in pts:
        if X == 0 and Y == 0:
            assert _compass(-X, Y, coeffs) == -1
            continue
        th = np.degrees(np.arctan2(Y, -X))                     # dz_dy, -dz_dx up to the common factor 1/8
        ref = 90.0 - th if th < 0 else (360.0 - th + 90.0 if th > 90.0 else 90.0 - th)
        got = float(_compass(np.float32(0.0) - np.float32(X) if X == 0 else -X, Y, coeffs))
        d = abs(got - ref)
        assert min(d, 360.0 - d) <= 1e-5 * abs(ref) + 1e-4, (X, Y, got, ref)


def _box_threshold(z):
    """NumPy statement of bs_threshold (box_stream.cu): 2^15 x the median |x| of the finite nonzero cells among
    128 fixed sample cells (the upper median when their number is even); 2^100 when there is none."""
    H, W = z.shape
    s = np.arange(128)
    a = np.abs(z[(2 * s + 1) * H // 256, (2 * ((79 * s) & 127) + 1) * W // 256].astype(np.float32))
    a = np.sort(a[np.isfinite(a) & (a > 0)])
    return np.float32(a[a.size // 2] * np.float32(32768.0)) if a.size else np.float32(2.0 ** 100)


def _box_running(z, kh, kw, w, seg_rows=40):
    """NumPy statement of box_stream_kernel (box_stream.cu): per column a float64 RUNNING sum V of the
    last kh rows (add the entering row, emit, subtract the leaving row -- restarted every `seg_rows`
    rows like the kernel's row segments), exceptional cells (NaN, infinite, or |v| >= the launch's cut-off
    `_box_threshold`) kept out of V and counted instead; horizontal window = difference of two inclusive
    prefixes of V; a window holding a NaN is NaN, one holding an infinite / exceptional cell is re-summed tap
    by tap in the reference's order, every other window is w * (running sum) + 0."""
    H, W = z.shape
    ry, rx = kh // 2, kw // 2
    huge = _box_threshold(z)
    zp = np.full((H + 2 * ry, W + 2 * rx), np.nan, np.float32)       # TMA out-of-raster fill
    zp[ry:ry + H, rx:rx + W] = z
    isnan = np.isnan(zp)
    with np.errstate(invalid="ignore"):
        big = ~isnan & ~(np.abs(zp) < huge)
    ordinary = np.where(isnan | big, 0.0, zp.astype(np.float64))
    out = np.empty((H, W), np.float32)
    for y0 in range(0, H, seg_rows):
        y1 = min(y0 + seg_rows, H)
        V = np.zeros(W + 2 * rx)
        Cn = np.zeros(W + 2 * rx, np.int64)
        Cb = np.zeros(W + 2 * rx, np.int64)
        for r in range(y1 - y0 + kh - 1):
            yy = y0 + r                        # row of the padded raster entering the window
            V = V + ordinary[yy]
            Cn += isnan[yy]
            Cb += big[yy]
            if r < kh - 1:
                continue
            y = y0 + r - (kh - 1)
            P = np.concatenate([[0.0], np.cumsum(V)])
            Pn = np.concatenate([[0], np.cumsum(Cn)])
            Pb = np.concatenate([[0], np.cumsum(Cb)])
            x = np.arange(W)
            win = P[x + kw] - P[x]
            res = (w * win + 0.0).astype(np.float32)
            nn, nb = Pn[x + kw] - Pn[x], Pb[x + kw] - Pb[x]
            res[nn > 0] = np.nan
            redo = np.nonzero((nn == 0) & (nb > 0))[0]
            if redo.size:                      # bs_direct: fma(w, v, acc) tap by tap
                res[redo] = o.convolve_2d_fma(zp[y:y + kh], np.full((kh, kw), w))[ry, redo + rx]
            out[y] = res
            V = V - ordinary[y0 + r - (kh - 1)]
            Cn -= isnan[y0 + r - (kh - 1)]
            Cb -= big[y0 + r - (kh - 1)]
    return out


@pytest.mark.parametrize("kh,kw", [(5, 5), (9, 9), (3, 7), (25, 3), (1, 5)])
def test_running_box_convolution_equals_tap_order_sums(kh, kw):
    """The running-sum form against the oracle's tap-order float64 accumulation: identical NaN masks,
    identical +-inf / huge results, finite results to float64 rounding -- including windows next to (but
    not containing) a FLT_MAX-style sentinel, which a summed-area table would have destroyed."""
    rng = np.random.default_rng(kh * 31 + kw)
    z = (terrain(rng, 70, 150) + 1e5).astype(np.float32)
    dirty = z.copy()
    dirty[10, 20] = np.nan
    dirty[40, 100] = np.inf
    dirty[55, 30] = np.float32(3.4028235e38)
    dirty[56, 31] = np.float32(-3.4028235e38)
    for w in (1.0 / (kh * kw), -0.37):
        for data in (z, dirty):
            ref = o.convolve_2d_fma(data, np.full((kh, kw), w), nthreads=4)   # the recompute's tap order
            got = _box_running(data, kh, kw, w)
            np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
            m = np.isfinite(ref) & (np.abs(ref) < 1e20)
            odd = ~m & ~np.isnan(ref)
            np.testing.assert_allclose(got[odd], ref[odd], rtol=1e-6)            # +-inf and huge windows
            np.testing.assert_allclose(got[m], ref[m], rtol=1e-6, atol=1e-6 * np.abs(ref[m]).max())


@pytest.mark.parametrize("field", ["terrain", "offset", "lognormal"])
@pytest.mark.parametrize("kh,kw", [(5, 5), (3, 9), (1, 7), (25, 25), (25, 3)])
def test_running_box_is_not_contaminated_by_large_cells(kh, kw, field):
    """A finite cell far above the data (a 1e20 fill value) must leave no rounding behind in the running column
    sums: every window without a NaN / inf / planted cell stays within 2 ulp32 + 2^-36 |w| kh kw M of the
    FMA-oracle's tap-order sum, for planted magnitudes from 2^24 M to FLT_MAX, both signs, single cells and
    3-row runs, at the model's segment starts and within kh rows of the raster's top and bottom.  With the
    former absolute 2^100 cut-off, 1e15 .. 1e29 entered V and left errors of up to the whole window."""
    rng = np.random.default_rng(kh * 100 + kw)
    H = 130
    z = box_magnitude_fields(rng, H, 60)[field]
    M = float(np.abs(z).max())
    rows = [0, 1, kh // 2, 40, 41, 80, 120, H - 1 - kh // 2, H - 2, H - 1]
    for value in box_planted_values(M):
        data, planted = box_plant(z, value, rows, rng)
        assert _box_threshold(data) <= 2.0 ** 15 * M
        for w in (1.0 / (kh * kw), -0.37):
            ref = o.convolve_2d_fma(data, np.full((kh, kw), w), nthreads=4)
            got = _box_running(data, kh, kw, w)
            box_window_errors(got, ref, planted, kh, kw, w, M, "%s %dx%d %g w=%g" % (field, kh, kw, value, w))


def _lane_sum_windows(v, rx):
    """NumPy statement of bs_lanesum / bs_cell (box_stream.cu, second-generation kernel): v[lane, j] = the
    float64 column sums a warp's 32 lanes hold (4 columns each).  Every lane forms the inclusive prefix
    and suffix of its own four values; the window of column 4 l + j is suffix[.] of the lane its left end
    falls in + prefix[.] of the lane its right end falls in + the totals of the whole lanes in between,
    every operand at a fixed lane distance (warp shuffles: a lane past the warp's end reads itself)."""
    q, m = divmod(rx, 4)
    lanes = np.arange(32)

    def frm(x, d):                       # __shfl_down_sync / __shfl_up_sync semantics
        src = lanes + d
        src = np.where((src < 0) | (src > 31), lanes, src)
        return x[src]

    pre = np.cumsum(v, axis=1)
    suf = np.empty_like(v)
    suf[:, 3] = v[:, 3]
    suf[:, 2] = v[:, 2] + suf[:, 3]
    suf[:, 1] = v[:, 1] + suf[:, 2]
    suf[:, 0] = pre[:, 3]
    tot = pre[:, 3]
    core, tl, tr = tot, np.zeros(32), np.zeros(32)
    if q == 2:
        core = (frm(tot, -1) + tot) + frm(tot, 1)
    if q == 3:
        pair = tot + frm(tot, 1)
        core = (frm(pair, -2) + pair) + frm(tot, 2)
    if q >= 1 and m > 0:
        tl, tr = frm(tot, -q), frm(tot, q)
    win = np.empty_like(v)
    for j in range(4):
        a, b = j - m, j + m
        if q == 0 and a >= 0 and b <= 3:
            assert a == 0 or b == 3
            win[:, j] = pre[:, b] if a == 0 else suf[:, a]
            continue
        dl, ia = -q - (1 if a < 0 else 0), (a + 4) & 3
        dh, ib = q + (1 if b >= 4 else 0), b & 3
        ends = frm(suf[:, ia], dl) + frm(pre[:, ib], dh)
        if q == 0:
            win[:, j] = ends + tot if (a < 0 and b >= 4) else ends
        else:
            full = core
            if a < 0:
                full = full + tl
            if b >= 4:
                full = full + tr
            win[:, j] = ends + full
    return win


@pytest.mark.parametrize("rx", range(1, 13))
def test_lane_sum_windows_equal_direct_window_sums(rx):
    """The shuffle algebra of the second-generation running-box kernel: for every lane that emits
    (4 * lane in [pad, 128 - pad), pad = rx rounded up to a multiple of 4) the lane-sum window equals the
    direct sum of the 2 rx + 1 columns (integers: exact in any order), and a NaN column (beyond the
    raster's edge: TMA fill) reaches exactly the windows that contain it -- no masking needed."""
    rng = np.random.default_rng(rx)
    cols = rng.integers(-1000, 1000, 128).astype(np.float64)
    pad = (rx + 3) // 4 * 4
    for nan_cols in ((), range(0, pad), range(128 - pad, 128), (pad + rx,)):
        c = cols.copy()
        c[list(nan_cols)] = np.nan
        with np.errstate(invalid="ignore"):
            win = _lane_sum_windows(c.reshape(32, 4), rx).reshape(128)
        x = np.arange(pad, 128 - pad)
        direct = np.array([c[i - rx:i + rx + 1].sum() for i in x])
        np.testing.assert_array_equal(win[x], direct)        # NaN == NaN positions included
    # the packed 16-bit pair counts go through the same algebra with unsigned adds
    cnt = rng.integers(0, 3, 128).astype(np.float64)
    win = _lane_sum_windows(cnt.reshape(32, 4), rx).reshape(128)
    x = np.arange(pad, 128 - pad)
    np.testing.assert_array_equal(win[x], np.array([cnt[i - rx:i + rx + 1].sum() for i in x]))


def test_focal_mean_division_by_count_is_correctly_rounded():
    """div_count9 (surface_ops.cuh) replaces the float64 division s / n (n = 1..9 valid cells) by
    q = s * (1/n), e = fma(-q, n, s), q + e * (1/n): with exact FMAs (emulated here with rationals)
    that is the correctly rounded quotient, i.e. bit-identical to np.nanmean's division."""
    from fractions import Fraction
    rng = np.random.default_rng(9)
    vals = np.concatenate([rng.standard_normal(4000) * 10.0 ** rng.integers(-8, 9, 4000),
                           rng.integers(-40000, 40000, 2000).astype(np.float64), [0.0, 1.0, 4000.0 * 9, 1e-300, 1e300]])
    bad = 0
    for s in vals:
        for n in range(1, 10):
            r = 1.0 / n
            q = s * r
            e = float(Fraction(s) - Fraction(q) * n)            # fma(-q, n, s): one rounding
            res = float(Fraction(e) * Fraction(r) + Fraction(q))  # fma(e, r, q): one rounding
            bad += res != s / n
    assert bad == 0


def test_running_box_mean_division_by_the_window_size_is_correctly_rounded():
    """bs_div_n (box_stream.cu, NaN-skipping mode = focal.apply mean over an all-ones window): the window sum
    divided by kh * kw as q = c * (1/n), q + fma(-q, n, c) * (1/n), for every window size the kernel serves
    (odd kh, kw <= 25).  With exact FMAs (rationals) that is the correctly rounded float64 quotient np.nanmean
    forms, so the float32 result cannot depend on which of the kernel's paths produced it."""
    from fractions import Fraction
    rng = np.random.default_rng(25)
    vals = np.concatenate([rng.standard_normal(300) * 10.0 ** rng.integers(-6, 9, 300),
                           rng.uniform(0, 4000 * 625, 300), [0.0, 1.0, 4000.0 * 625, 1e-300, 1e300]])
    sizes = sorted({kh * kw for kh in range(1, 26, 2) for kw in range(3, 26, 2)})
    bad = 0
    for c in vals:
        for n in sizes:
            inv = 1.0 / n
            q = c * inv
            r = float(Fraction(c) - Fraction(q) * n)               # fma(-q, n, c): one rounding
            res = float(Fraction(r) * Fraction(inv) + Fraction(q))  # fma(r, inv, q): one rounding
            bad += res != c / n
    assert bad == 0


@pytest.mark.parametrize("az,alt", [(225.0, 25.0), (0.0, 90.0), (90.0, 1.0), (315.0, 60.0)])
def test_hillshade_closed_form_equals_the_trig_chain(az, alt):
    """HillshadeOp (surface_ops.cuh) evaluates hillshade.py:20-35 -- np.gradient, atan, atan2, sin, cos --
    as [sin(alt) + cos(alt) (cos A gy - sin A gx)] / sqrt(1 + gx^2 + gy^2), A = azimuth_rad - pi/2, in float32
    with the doubled gradients gx2 = 2 gx, gy2 = 2 gy: no transcendental per cell.  Same numbers as the
    oracle's trig chain (the float32 noise of either form is ~1e-7)."""
    rng = np.random.default_rng(int(az + alt))
    z = terrain(rng, 60, 90)
    ref = o.hillshade(z, az, alt, nthreads=2).astype(np.float64)
    azr = (360.0 - az) * np.pi / 180.0
    altr = alt * np.pi / 180.0
    a_ = azr - np.pi / 2.0
    s0, cy, cx = np.float32(np.sin(altr)), np.float32(0.5 * np.cos(altr) * np.cos(a_)), np.float32(0.5 * np.cos(altr) * np.sin(a_))
    gx2 = (z[2:, 1:-1] - z[:-2, 1:-1]).astype(np.float32)      # 2 * d/drow
    gy2 = (z[1:-1, 2:] - z[1:-1, :-2]).astype(np.float32)      # 2 * d/dcol
    q = (gx2 * gx2 + gy2 * gy2).astype(np.float32)
    rinv = (1.0 / np.sqrt((np.float32(0.25) * q + np.float32(1.0)).astype(np.float64))).astype(np.float32)
    num = (cy * gy2 + (-cx * gx2 + s0)).astype(np.float32)
    got = (np.float32(0.5) * num * rinv + np.float32(0.5)).astype(np.float64)
    np.testing.assert_allclose(got, ref[1:-1, 1:-1], rtol=1e-5, atol=1e-6)
    assert np.isnan(ref[0]).all() and np.isnan(ref[:, 0]).all()


def test_slope_sum_of_squares_form():
    """SlopeOp: X = 8 csx dz_dx and Y = 8 csy dz_dy are exact in float64; the kernel forms
    p = ky^2 ((X kx / ky)^2 + Y^2), rounds it to float32 once and takes atan(sqrt(p)) in float32."""
    rng = np.random.default_rng(12)
    z = terrain(rng, 50, 70)
    for csx, csy in ((30.0, 30.0), (10.0, 25.0), (1.0, -1.0)):
        ref = o.slope(z, csx, csy, nthreads=2).astype(np.float64)
        zz = z.astype(np.float64)
        # slope.py:64-71: a,b,c = row y+1; g,h,i = row y-1
        X = (zz[2:, 2:] + 2 * zz[1:-1, 2:] + zz[:-2, 2:]) - (zz[2:, :-2] + 2 * zz[1:-1, :-2] + zz[:-2, :-2])
        Y = (zz[:-2, :-2] + 2 * zz[:-2, 1:-1] + zz[:-2, 2:]) - (zz[2:, :-2] + 2 * zz[2:, 1:-1] + zz[2:, 2:])
        kx, ky = 1.0 / (8.0 * csx), 1.0 / (8.0 * csy)
        xs = X * (kx / ky)
        p = (xs * xs + Y * Y).astype(np.float32) * np.float32(ky * ky)
        got = np.degrees(np.arctan(np.sqrt(p.astype(np.float64)))) * (57.29578 / (180.0 / np.pi))
        np.testing.assert_allclose(got, ref[1:-1, 1:-1], rtol=1e-5, atol=1e-6)


def test_order_preserving_float_keys_of_the_zonal_table():
    """zh_fkey / zh_funkey (zonal_hash.cu): int32 keys whose signed order is the float order, so the
    per-CTA min / max are native integer atomics; the map is its own inverse."""
    rng = np.random.default_rng(5)
    f = np.concatenate([rng.standard_normal(5000).astype(np.float32) * np.float32(10.0) ** rng.integers(-30, 30, 5000),
                        np.array([0.0, -0.0, np.inf, -np.inf, 1e-45, -1e-45, 3.4e38, -3.4e38], np.float32)]).astype(np.float32)
    b = f.view(np.int32)
    key = b ^ ((b >> 31) & np.int32(0x7fffffff))
    back = (key ^ ((key >> 31) & np.int32(0x7fffffff))).view(np.float32)
    np.testing.assert_array_equal(back.view(np.int32), b)
    order = np.argsort(key, kind="stable")
    assert (np.diff(f[order].astype(np.float64)) >= 0).all()
    assert key[f == np.inf][0] == np.int32(0x7f800000) and (key[np.isfinite(f)] < np.int32(0x7f800000)).all()


def _compile_lane_sum_templates(tmp_path):
    """The device templates bs_from / bs_cell / bs_lanesum, cut out of box_stream.cu verbatim and compiled for the
    HOST with a 32-lane value type whose shuffles have the hardware's semantics (a lane past the warp's end
    reads itself): every compile-time radius is instantiated from the shipped source, not from a restatement."""
    import ctypes
    import subprocess
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "xarray-spatial_b200", "csrc",
                            "box_stream.cu")).read()
    a = src.index("// the value lane (l + D) holds")
    b = src.index("__device__ __forceinline__ uint32_t bs_bits(int n)")
    body = src[a:b]
    host = r"""
#include <cmath>
#define __device__
#define __forceinline__ inline
struct Lanes {
    double v[32];
    Lanes() {}
    Lanes(double x) { for (int i = 0; i < 32; ++i) v[i] = x; }
};
inline Lanes operator+(const Lanes &a, const Lanes &b) { Lanes r; for (int i = 0; i < 32; ++i) r.v[i] = a.v[i] + b.v[i]; return r; }
inline Lanes __shfl_down_sync(unsigned, const Lanes &x, int d) { Lanes r; for (int l = 0; l < 32; ++l) r.v[l] = l + d <= 31 ? x.v[l + d] : x.v[l]; return r; }
inline Lanes __shfl_up_sync(unsigned, const Lanes &x, int d) { Lanes r; for (int l = 0; l < 32; ++l) r.v[l] = l - d >= 0 ? x.v[l - d] : x.v[l]; return r; }
// names of the float64-only branch of bs_from (discarded for Lanes, but parsed)
int __double2loint(double); int __double2hiint(double); double __hiloint2double(int, int);
int __shfl_down_sync(unsigned, int, int); int __shfl_up_sync(unsigned, int, int);
""" + body + r"""
template <int RX> static void run1(const double *cols, double *out) {
    Lanes v[1][4], w[1][4];
    for (int l = 0; l < 32; ++l) for (int j = 0; j < 4; ++j) v[0][j].v[l] = cols[4 * l + j];
    bs_lanesum<RX, 1, Lanes>(v, w);
    for (int l = 0; l < 32; ++l) for (int j = 0; j < 4; ++j) out[4 * l + j] = w[0][j].v[l];
}
extern "C" int lane_sum(int rx, const double *cols, double *out) {
    switch (rx) {
        case 1: run1<1>(cols, out); break;   case 2: run1<2>(cols, out); break;   case 3: run1<3>(cols, out); break;
        case 4: run1<4>(cols, out); break;   case 5: run1<5>(cols, out); break;   case 6: run1<6>(cols, out); break;
        case 7: run1<7>(cols, out); break;   case 8: run1<8>(cols, out); break;   case 9: run1<9>(cols, out); break;
        case 10: run1<10>(cols, out); break; case 11: run1<11>(cols, out); break; case 12: run1<12>(cols, out); break;
        default: return 1;
    }
    return 0;
}
"""
    cpp = os.path.join(str(tmp_path), "lane_sum_host.cpp")
    so = os.path.join(str(tmp_path), "lane_sum_host.so")
    open(cpp, "w").write(host)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-o", so, cpp])
    lib = ctypes.CDLL(so)
    lib.lane_sum.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    return lib


def test_shipped_lane_sum_templates_on_the_host(tmp_path):
    """Every radius 1..12 of the SHIPPED templates (compiled for the host, see above) against direct window sums,
    with NaN columns beyond either edge of the strip: this is the code the GPU runs, minus the hardware."""
    lib = _compile_lane_sum_templates(tmp_path)
    rng = np.random.default_rng(77)
    for rx in range(1, 13):
        pad = (rx + 3) // 4 * 4
        x = np.arange(pad, 128 - pad)
        for nan_cols in ((), range(0, pad), range(128 - pad, 128), (pad + rx,)):
            cols = rng.integers(-1000, 1000, 128).astype(np.float64)
            cols[list(nan_cols)] = np.nan
            out = np.empty(128)
            assert lib.lane_sum(rx, cols.ctypes.data, out.ctypes.data) == 0
            with np.errstate(invalid="ignore"):
                direct = np.array([cols[i - rx:i + rx + 1].sum() for i in x])
            np.testing.assert_array_equal(out[x], direct, err_msg="radius %d" % rx)


def _lane_sum_windows_wide(v, rx):
    """NumPy statement of bw_lanesum / bw_cell of the WIDE variant of the running box (a tuning note, not built:
    scripts/tune/box_stream_wide_variant.cu.txt -- measured slower than the shipped kernel): 8 columns per lane, 256 per warp,
    radius <= 12.  Same algebra as _lane_sum_windows: suffix of the lane the window starts in + prefix of the
    lane it ends in + the totals of whole lanes in between; a window inside one lane is summed directly."""
    q, m = divmod(rx, 8)
    lanes = np.arange(32)

    def frm(x, d):
        src = lanes + d
        src = np.where((src < 0) | (src > 31), lanes, src)
        return x[src]

    pre = np.cumsum(v, axis=1)
    suf = np.empty_like(v)
    suf[:, 7] = v[:, 7]
    for j in range(6, 0, -1):
        suf[:, j] = v[:, j] + suf[:, j + 1]
    suf[:, 0] = pre[:, 7]
    tot = pre[:, 7]
    tl, tr = (frm(tot, -1), frm(tot, 1)) if (q == 1 and m > 0) else (np.zeros(32), np.zeros(32))
    win = np.empty_like(v)
    for j in range(8):
        a, b = j - m, j + m
        if q == 0 and a >= 0 and b <= 7:
            if a == 0:
                win[:, j] = pre[:, b]
            elif b == 7:
                win[:, j] = suf[:, a]
            else:
                acc = v[:, a].copy()
                for c in range(a + 1, b + 1):
                    acc = acc + v[:, c]
                win[:, j] = acc
            continue
        dl, ia = -q - (1 if a < 0 else 0), (a + 8) & 7
        dh, ib = q + (1 if b >= 8 else 0), b & 7
        ends = frm(suf[:, ia], dl) + frm(pre[:, ib], dh)
        if q == 0:
            win[:, j] = ends + tot if (a < 0 and b >= 8) else ends
        else:
            full = tot
            if a < 0:
                full = full + tl
            if b >= 8:
                full = full + tr
            win[:, j] = ends + full
    return win


@pytest.mark.parametrize("rx", range(1, 13))
def test_wide_lane_sum_windows_equal_direct_window_sums(rx):
    """The wide variant's shuffle algebra (8 columns per lane): every column whose float4 half emits (half start
    in [pad, 256 - pad), pad = rx rounded up to a multiple of 4) gets the direct sum of its 2 rx + 1 columns, and
    NaN columns beyond the raster's edge -- whole lanes, or ONE half of a lane -- reach exactly the windows that
    contain them."""
    rng = np.random.default_rng(100 + rx)
    cols = rng.integers(-1000, 1000, 256).astype(np.float64)
    pad = (rx + 3) // 4 * 4
    x = np.arange(pad, 256 - pad)
    for nan_cols in ((), range(0, pad), range(256 - pad, 256), range(0, 4), range(0, 12), range(252, 256), (pad + rx,)):
        c = cols.copy()
        c[list(nan_cols)] = np.nan
        with np.errstate(invalid="ignore"):
            win = _lane_sum_windows_wide(c.reshape(32, 8), rx).reshape(256)
        direct = np.array([c[i - rx:i + rx + 1].sum() for i in x])
        np.testing.assert_array_equal(win[x], direct)
    cnt = rng.integers(0, 3, 256).astype(np.float64)
    win = _lane_sum_windows_wide(cnt.reshape(32, 8), rx).reshape(256)
    np.testing.assert_array_equal(win[x], np.array([cnt[i - rx:i + rx + 1].sum() for i in x]))


def _pair_counts_two_runs(zones, values, nodata=None):
    """NumPy statement of zonal_pair_kernel's bookkeeping (zonal_hash.cu): a lane walks down its 4 columns and
    keeps TWO open runs (zone, value, count); a cell whose pair is one of them just counts, a third pair evicts
    the run used less recently into the table.  A 4-row batch is "clean" when every cell lies in the zone of
    the run used last and holds one of the two values whose runs are in that zone -- then the batch is counted
    by value compares alone (an invalid cell matches neither value, so validity needs no test there)."""
    H, W = zones.shape
    table = {}

    def merge(z, v, c):
        if c:
            table[(int(z), float(v))] = table.get((int(z), float(v)), 0) + int(c)

    for x0 in range(0, W, 4):
        z0 = z1 = 0
        v0 = v1 = np.float32(np.nan)
        c0 = c1 = 0
        last1 = False
        for y0 in range(0, H, 4):
            zb, vb = zones[y0:y0 + 4, x0:x0 + 4], values[y0:y0 + 4, x0:x0 + 4]
            zc = z1 if last1 else z0
            m0 = int((vb == v0).sum()) if z0 == zc else 0
            m1 = int((vb == v1).sum()) if z1 == zc else 0
            if zb.shape == (4, 4) and (zb == zc).all() and m0 + m1 == 16:
                c0, c1 = c0 + m0, c1 + m1
                last1 = bool(z1 == zc and vb[3, 3] == v1)
                continue
            for zk, fr in zip(zb.ravel(), vb.ravel()):        # row-major inside the batch, like the kernel
                f = np.float32(fr + np.float32(0.0))
                if not np.isfinite(f) or (nodata is not None and f == nodata):
                    continue
                if zk == z0 and f == v0:
                    c0, last1 = c0 + 1, False
                elif zk == z1 and f == v1:
                    c1, last1 = c1 + 1, True
                elif last1:
                    merge(z0, v0, c0)
                    z0, v0, c0, last1 = zk, f, 1, False
                else:
                    merge(z1, v1, c1)
                    z1, v1, c1, last1 = zk, f, 1, True
        merge(z0, v0, c0)
        merge(z1, v1, c1)
    return table


def test_two_open_runs_count_every_pair_exactly_once():
    """The pair histogram behind `majority` / `crosstab`: whatever the flip-flop pattern between classes, zone
    boundaries, NaN / inf / nodata cells and -0.0, the two-run bookkeeping counts every valid (zone, value)
    pair exactly once (compared with a direct histogram)."""
    rng = np.random.default_rng(2)
    H, W = 64, 24
    for trial in range(6):
        base = np.cumsum(rng.standard_normal((H, W)) * 0.7, axis=0)          # smooth down the columns: long runs
        values = np.floor(base + rng.standard_normal((H, W)) * (0.2 + 0.2 * trial)).astype(np.float32)   # + flip-flops
        zones = (np.arange(H)[:, None] // (8 + trial) * 3 + np.arange(W)[None, :] // 5).astype(np.int32)
        values[rng.random((H, W)) < 0.03] = np.nan
        values[5, 7] = np.inf
        values[9, 3] = np.float32(-0.0)
        nodata = np.float32(2.0) if trial % 2 else None
        got = _pair_counts_two_runs(zones, values, nodata)
        ok = np.isfinite(values) & ((values != nodata) if nodata is not None else True)
        ref = {}
        for z, v in zip(zones[ok], values[ok]):
            k = (int(z), float(v + np.float32(0.0)))
            ref[k] = ref.get(k, 0) + 1
        assert got == ref


def test_shipped_division_and_float_keys_on_the_host(tmp_path):
    """Two more device helpers cut out of the shipped sources and compiled for the host: bs_div_n (box_stream.cu;
    the window sum divided by the window size) against the float64 division, and zh_fkey / zh_funkey
    (zonal_hash.cu; order-preserving int32 keys of float32 values, so that min / max are native integer atomics)
    against float ordering and a bit-exact round trip."""
    import ctypes
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    box = open(os.path.join(root, "xarray-spatial_b200", "csrc", "box_stream.cu")).read()
    zh = open(os.path.join(root, "xarray-spatial_b200", "csrc", "zonal_hash.cu")).read()
    a = box.index("__device__ __forceinline__ double bs_div_n(")
    div_src = box[a:box.index("}", box.index("return fma(", a)) + 1]
    a = zh.index("__device__ __forceinline__ int zh_fkey(float f)")
    key_src = zh[a:zh.index("template <typename VT> struct ZhMinMax")]
    host = r"""
#include <cmath>
#include <cstring>
#define __device__
#define __forceinline__ inline
static inline int __float_as_int(float f) { int i; std::memcpy(&i, &f, 4); return i; }
static inline float __int_as_float(int i) { float f; std::memcpy(&f, &i, 4); return f; }
""" + div_src + "\n" + key_src + r"""
extern "C" double div_n(double c, double n) { return bs_div_n(c, n, 1.0 / n); }
extern "C" int fkey(float f) { return zh_fkey(f); }
extern "C" float funkey(int k) { return zh_funkey(k); }
"""
    cpp, so = os.path.join(str(tmp_path), "h.cpp"), os.path.join(str(tmp_path), "h.so")
    open(cpp, "w").write(host)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, cpp])
    lib = ctypes.CDLL(so)
    lib.div_n.restype, lib.div_n.argtypes = ctypes.c_double, [ctypes.c_double, ctypes.c_double]
    lib.fkey.restype, lib.fkey.argtypes = ctypes.c_int, [ctypes.c_float]
    lib.funkey.restype, lib.funkey.argtypes = ctypes.c_float, [ctypes.c_int]
    rng = np.random.default_rng(5)
    sizes = sorted({kh * kw for kh in range(1, 26, 2) for kw in range(3, 26, 2)})
    for c in np.concatenate([rng.uniform(0, 4000 * 625, 200), rng.standard_normal(200) * 10.0 ** rng.integers(-6, 9, 200)]):
        for n in sizes:
            assert lib.div_n(float(c), float(n)) == c / n, (c, n)
    vals = np.concatenate([rng.standard_normal(2000).astype(np.float32) * np.float32(10.0) ** rng.integers(-20, 20, 2000).astype(np.float32),
                           np.array([0.0, -0.0, np.inf, -np.inf, 1e-45, -1e-45, 3.4028235e38, -3.4028235e38], np.float32)])
    keys = np.array([lib.fkey(ctypes.c_float(float(v))) for v in vals], np.int64)
    order = np.argsort(vals, kind="stable")
    strictly = np.diff(vals[order]) > 0                           # float order == key order (-0.0 and 0.0 compare equal
    assert (np.diff(keys[order])[strictly] > 0).all()             # and may keep either key: the sign of a zero min / max)
    back = np.array([lib.funkey(int(k)) for k in keys], np.float32)
    np.testing.assert_array_equal(back.view(np.int32), vals.view(np.int32))   # bit-exact round trip

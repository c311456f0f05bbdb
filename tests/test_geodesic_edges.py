"""Geodesic slope / aspect (csrc/geodesic.cu) against an extended-precision statement of the reference.

T, below, is geodesic.py:40-172 written in NumPy over np.longdouble: ECEF coordinates, the centre cell's
East/North/Up frame, the curvature correction u += (e^2 + n^2) / 2R and the centred normal equations, in the
reference's form.  The regular-grid kernel computes the same plane in another algebraic form (per-row and
per-column trig tables, the rotation folded, uncentred sums) and ends in a float32 atan / compass polynomial.
Every kernel cell is held to

    |kernel - T| <= 8 ulp32(T) + 4 |oracle - T| + 1e-8 degrees

(aspect: circular difference, ulp32(max(T, 1))).  The 8 ulps are the float32 tail (bounded on the CPU below
from the header's coefficients); the second term grants the kernel the float64 rounding the reference's own
arithmetic makes where double precision cancels (a flat surface, 1e-6 degree cells); the last term covers
slopes far below a float32 ulp of anything.  NaN and flat (-1) masks must equal the oracle's exactly.

The CPU tests pin T to the oracle and the tail to the bound; the GPU tests run the public slope / aspect
over latitudes, longitudes, spacings, coordinate forms, cell types, z units, NaNs, compass directions,
shapes, launch sizes and memory layouts."""
import numpy as np
import pytest

import oracle as o
from test_kernel_algebra import _atan_coeffs, _compass

L = np.longdouble
# x86-64 extended (64-bit significand) or IEEE quad: T must be far more precise than the float64 it checks
assert np.finfo(np.longdouble).eps <= 2.0 ** -63, "np.longdouble is no wider than float64 on this platform"

A2 = L(6378137.0) ** 2
B2 = L(6356752.314245) ** 2
INV_2R = L(1) / (L(2) * L(6370994.884953014))
D2R = np.arctan(L(1)) / L(45)
R2D = L(45) / np.arctan(L(1))
S1 = 1.0 / 3600.0                                  # one arcsecond in degrees
R_M = 6371000.0


def ulp32(x):
    return np.spacing(np.abs(np.asarray(x, np.float64)).astype(np.float32)).astype(np.float64)


# ------------------------------------------------------------------------------------------- the statement
def _fit(h, la, lo, zf):
    """(A, B) of every interior cell of one block of rows (geodesic.py:40-131), longdouble."""
    H, W = h.shape
    h = h.astype(L) * L(zf)
    la, lo = la.astype(L) * D2R, lo.astype(L) * D2R
    sl, cl, so, co = np.sin(la), np.cos(la), np.sin(lo), np.cos(lo)
    N = A2 / np.sqrt(A2 * cl * cl + B2 * sl * sl)
    X, Y, Z = (N + h) * cl * co, (N + h) * cl * so, (B2 / A2 * N + h) * sl
    c = (slice(1, H - 1), slice(1, W - 1))
    ex, ey = -so[c], co[c]
    nx, ny, nz = -sl[c] * co[c], -sl[c] * so[c], cl[c]
    ux, uy, uz = cl[c] * co[c], cl[c] * so[c], sl[c]
    E, Nn, U, bad = [], [], [], np.zeros((H - 2, W - 2), bool)
    for dy in range(3):
        for dx in range(3):
            k = (slice(dy, H - 2 + dy), slice(dx, W - 2 + dx))
            ddx, ddy, ddz = X[k] - X[c], Y[k] - Y[c], Z[k] - Z[c]
            e = ddx * ex + ddy * ey
            n = ddx * nx + ddy * ny + ddz * nz
            u = ddx * ux + ddy * uy + ddz * uz + (e * e + n * n) * INV_2R
            E.append(e), Nn.append(n), U.append(u)
            bad |= np.isnan(h[k])
    E, Nn, U = np.array(E), np.array(Nn), np.array(U)
    E, Nn, U = E - E.mean(0), Nn - Nn.mean(0), U - U.mean(0)
    See, Snn, Sen = (E * E).sum(0), (Nn * Nn).sum(0), (E * Nn).sum(0)
    Seu, Snu = (E * U).sum(0), (Nn * U).sum(0)
    det = See * Snn - Sen * Sen
    flat = np.abs(det) < 1e-30                       # degenerate -> flat (geodesic.py:124-125)
    with np.errstate(divide="ignore", invalid="ignore"):
        A = np.where(flat, L(0), (Seu * Snn - Snu * Sen) / det)
        B = np.where(flat, L(0), (Snu * See - Seu * Sen) / det)
    A[bad], B[bad] = np.nan, np.nan                  # a NaN elevation in the window (geodesic.py:66-68)
    return A, B


def truth(z, lat2, lon2, zf=1.0, rows=256):
    """T: (slope, aspect, |(A, B)|) over the raster in longdouble, NaN ring, in blocks of centre rows."""
    H, W = z.shape
    sl, asp, mag = (np.full((H, W), np.nan, L) for _ in range(3))
    if H < 3 or W < 3:
        return sl, asp, mag
    for y0 in range(1, H - 1, rows):
        y1 = min(H - 1, y0 + rows)
        A, B = _fit(z[y0 - 1:y1 + 1], lat2[y0 - 1:y1 + 1], lon2[y0 - 1:y1 + 1], zf)
        m = np.sqrt(A * A + B * B)
        a = np.arctan2(-A, -B) * R2D
        a = np.where(a < 0, a + 360, a)
        a = np.where(a >= 360, a - 360, a)
        sl[y0:y1, 1:-1] = np.arctan(m) * R2D         # geodesic.py:141-142
        asp[y0:y1, 1:-1] = np.where(m < 1e-7, L(-1), a)   # geodesic.py:155-166
        mag[y0:y1, 1:-1] = m
    return sl, asp, mag


def _b2(lat, lon, shape):
    if np.ndim(lat) == 2:
        return np.asarray(lat, np.float64), np.asarray(lon, np.float64)
    return (np.ascontiguousarray(np.broadcast_to(np.asarray(lat, np.float64)[:, None], shape)),
            np.ascontiguousarray(np.broadcast_to(np.asarray(lon, np.float64)[None, :], shape)))


def expect(z, lat, lon, zf=1.0):
    """T and the oracle on the float64 values of `z` (what the product computes on)."""
    z64 = np.asarray(z).astype(np.float64)
    la2, lo2 = _b2(lat, lon, z64.shape)
    ts, ta, mag = truth(z64, la2, lo2, zf)
    n = o.max_threads()
    return dict(slope=ts, aspect=ta, mag=mag, o_slope=o.geodesic(z64, la2, lo2, z_factor=zf, nthreads=n),
                o_aspect=o.geodesic(z64, la2, lo2, z_factor=zf, aspect=True, nthreads=n))


def _err(got, T, ref, aspect):
    """(|got - T|, allowed) on the cells with a value (not NaN, not -1)."""
    m = np.isfinite(ref) & (ref != -1 if aspect else True)
    g, t, r = got[m].astype(np.float64), T[m], ref[m].astype(np.float64)
    d = np.abs(g.astype(L) - t).astype(np.float64)
    dr = np.abs(r.astype(L) - t).astype(np.float64)
    scale = np.maximum(t.astype(np.float64), 1.0) if aspect else t.astype(np.float64)
    if aspect:
        d, dr = np.minimum(d, 360.0 - d), np.minimum(dr, 360.0 - dr)
    return d, 8.0 * ulp32(scale) + 4.0 * dr + 1e-8, ulp32(scale)


WORST = {}


def check(got, ex, what, aspect=False):
    """The kernel's output `got` against T and the oracle in `ex`; returns the worst error in float32 ulps."""
    got = np.asarray(got)
    assert got.dtype == np.float32 and got.shape == ex["slope"].shape, (got.dtype, got.shape)
    key = "aspect" if aspect else "slope"
    T, ref = ex[key], ex["o_" + key]
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref), err_msg=what + ": NaN mask differs from the oracle")
    np.testing.assert_array_equal(np.isnan(T), np.isnan(ref), err_msg=what + ": NaN mask of T differs")
    if aspect:
        np.testing.assert_array_equal(got == -1, ref == -1, err_msg=what + ": flat mask differs from the oracle")
        np.testing.assert_array_equal(T == -1, ref == -1, err_msg=what + ": flat mask of T differs")
    d, tol, u = _err(got, T, ref, aspect)
    bad = d > tol
    if bad.any():
        i = np.argmax(d - tol)
        raise AssertionError("%s %s: %d of %d cells outside the bound; worst |kernel - T| = %.3g deg = %.1f ulp32 "
                             "(allowed %.3g)" % (what, key, bad.sum(), d.size, d[i], d[i] / u[i], tol[i]))
    big = T[np.isfinite(ref) & (ref != -1 if aspect else True)].astype(np.float64) >= 1e-4   # ulps of a slope
    worst = (float((d / u)[big].max()) if big.any() else 0.0, float(d.max()) if d.size else 0.0)   # of ~0 mean little
    prev = WORST.get(key, (0.0, 0.0))
    WORST[key] = (max(prev[0], worst[0]), max(prev[1], worst[1]))
    print("geodesic %-40s %-6s max %6.2f ulp32  %.3g deg" % (what, key, worst[0], worst[1]))
    return worst[0]


# ------------------------------------------------------------------------------------------- fixtures
def axis(v0, step, n, rng=None):
    """n coordinates from v0 by `step`; with `rng`, each step is drawn from 0.5 .. 1.5 times `step`."""
    s = np.full(n - 1, float(step)) if rng is None else step * rng.uniform(0.5, 1.5, n - 1)
    return v0 + np.concatenate([[0.0], np.cumsum(s)])


def surface(lat2, lon2, seed, grade=1.0):
    """Smooth elevation (m) over the cells: a tilted plane and three sinusoids laid out in local metres with a
    wavelength of about ten cells, so slopes span about 0.01 .. 60 degrees whatever the cell size."""
    rng = np.random.default_rng(seed)
    lat2, lon2 = np.asarray(lat2, np.float64), np.asarray(lon2, np.float64)
    dlon = (lon2 - lon2[:1, :1] + 180.0) % 360.0 - 180.0
    y = np.radians(lat2 - lat2[:1, :1]) * R_M
    x = np.radians(dlon) * R_M * np.cos(np.radians(lat2))
    cell = max(np.nanmedian(np.abs(np.diff(y, axis=0))) if y.shape[0] > 1 else 0.0,
               np.nanmedian(np.abs(np.diff(x, axis=1))) if x.shape[1] > 1 else 0.0, 1e-9)
    lam = 10.0 * cell
    z = grade * (0.05 * x + 0.03 * y)
    for _ in range(3):
        th, ph = rng.uniform(0, 2 * np.pi, 2)
        k = 2 * np.pi / (lam * rng.uniform(0.7, 1.5))
        z += grade * 0.45 / k * np.sin(k * (x * np.cos(th) + y * np.sin(th)) + ph)
    return z + 500.0


def regular(lat, lon, seed=0, grade=1.0):
    la2, lo2 = _b2(lat, lon, (len(lat), len(lon)))
    return dict(z=surface(la2, lo2, seed, grade), lat=np.asarray(lat, np.float64), lon=np.asarray(lon, np.float64))


def curvilinear(kind, H=40, W=52, lat0=46.0, lon0=7.0, step=S1, seed=0):
    """2-D coordinates: the 1-D grid rotated by 20 degrees, or perturbed by 0.2 cell per coordinate."""
    i, j = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    if kind == "rotated":
        t = np.radians(20.0)
        lat2 = lat0 - step * (i * np.cos(t) - j * np.sin(t))
        lon2 = lon0 + step * (i * np.sin(t) + j * np.cos(t))
    else:
        rng = np.random.default_rng(seed + 7)
        lat2 = lat0 - step * i + 0.2 * step * rng.uniform(-1, 1, (H, W))
        lon2 = lon0 + step * j + 0.2 * step * rng.uniform(-1, 1, (H, W))
    return dict(z=surface(lat2, lon2, seed), lat=lat2, lon=lon2)


def _antimeridian(wrapped):
    lon = axis(179.99, S1, 52) - 0.5 * 51 * S1 + 0.01
    if wrapped:
        lon = np.where(lon > 180.0, lon - 360.0, lon)
    lat = axis(50.0, -S1, 40)
    c = regular(lat, np.where(lon > 180.0, lon - 360.0, lon), seed=3)   # the same surface for both forms
    c["lon"] = lon
    return c


CASES = {
    "46N_descending_1s": lambda: regular(axis(46.0, -S1, 40), axis(7.0, S1, 52)),
    "equator_straddle_1s": lambda: regular(axis(0.0055, -S1, 40), axis(-60.0, S1, 52), seed=1),
    "60S_ascending_3s": lambda: regular(axis(-60.0, 3 * S1, 40), axis(-70.0, 3 * S1, 52), seed=2),
    "north_pole_row": lambda: regular(axis(90.0, -S1, 40), axis(10.0, 2.0, 52), seed=4),
    "south_pole_row": lambda: regular(axis(-90.0 + 39 * S1, -S1, 40), axis(-30.0, 2.0, 52), seed=5),
    "antimeridian_wrapped": lambda: _antimeridian(True),
    "antimeridian_0_360": lambda: _antimeridian(False),
    "spacing_1e-6deg": lambda: regular(axis(30.0, -1e-6, 40), axis(10.0, 1e-6, 52), seed=6),
    "spacing_30s": lambda: regular(axis(46.0, -30 * S1, 40), axis(7.0, 30 * S1, 52), seed=7),
    "spacing_1deg": lambda: regular(axis(40.0, -1.0, 40), axis(-20.0, 1.0, 52), seed=8),
    "irregular_1s": lambda: regular(axis(46.0, -S1, 40, np.random.default_rng(9)),
                                    axis(7.0, S1, 52, np.random.default_rng(10)), seed=9),
    "irregular_30s": lambda: regular(axis(-20.0, 30 * S1, 40, np.random.default_rng(11)),
                                     axis(120.0, 30 * S1, 52, np.random.default_rng(12)), seed=10),
    "rotated_2d": lambda: curvilinear("rotated"),
    "perturbed_2d": lambda: curvilinear("perturbed", lat0=-33.0, lon0=151.0, step=3 * S1, seed=1),
}

CANCELS = {"spacing_1e-6deg"}      # fixtures on which float64 cancels (see the first CPU test)


@pytest.fixture(scope="module")
def cases():
    out = {}
    for name, make in CASES.items():
        c = make()
        for dt in (np.float64, np.float32):
            z = c["z"].astype(dt)
            out[name, dt] = dict(c, z=z, ex=expect(z, c["lat"], c["lon"]))
    return out


# ------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("name", sorted(CASES))
def test_extended_statement_agrees_with_the_oracle(cases, name):
    """T and the float64 oracle agree to a float32 ulp on every well-conditioned fixture: both state
    geodesic.py, so a larger gap would be a wrong statement or an ill-conditioned fixture.  On 1e-6 degree
    cells float64 ECEF coordinates (~6.4e6 m) keep ~1e-9 m of 0.1 m offsets, and the oracle is off by tens
    of ulps; the bound's |oracle - T| term is there for that.  No fixture has |(A, B)| within a factor of 3
    of the 1e-7 flat threshold, and the slopes cover about 1 .. 50 degrees."""
    for dt in (np.float64, np.float32):
        ex = cases[name, dt]["ex"]
        for key in ("slope", "aspect"):
            T, ref = ex[key], ex["o_" + key]
            np.testing.assert_array_equal(np.isnan(T), np.isnan(ref))
            d, _, u = _err(ref, T, ref, key == "aspect")
            print("%s %s %s: oracle vs T, max %.2f ulp32" % (name, dt.__name__, key, (d / u).max()))
            assert (d <= (64 if name in CANCELS else 1) * u).all(), (name, key, (d / u).max())
        mag = ex["mag"][np.isfinite(ex["mag"])].astype(np.float64)
        assert not ((mag > 1e-7 / 3) & (mag < 3e-7)).any()
        s = ex["o_slope"][np.isfinite(ex["o_slope"])]
        assert s.min() < 2.0 and s.max() > 40.0, (name, s.min(), s.max())


def _tail_slope(m2, rs):
    """atan_sqrt_deg (common.cuh) in float32 with the reciprocal square root `rs(p)`."""
    c = _atan_coeffs()
    p = np.asarray(m2, np.float64).astype(np.float32)
    r = rs(np.maximum(p, np.float32(1e-30)))
    big = p > 1
    a = np.where(big, -r, (p * r).astype(np.float32)).astype(np.float32)
    off = np.where(big, np.float32(np.float32(1.57079632679489662) * np.float32(57.29578)), np.float32(0))
    z = (a * a).astype(np.float32)
    q = np.full_like(z, np.float32(c[0]) * np.float32(57.29578))
    for k in c[1:]:
        q = (q.astype(np.float64) * z + np.float64(np.float32(k) * np.float32(57.29578))).astype(np.float32)
    return (a.astype(np.float64) * q + off).astype(np.float32)


def _rsqrt(rel):
    """float32 reciprocal square root with relative error `rel` (rsqrt.approx is within 2^-22.9)."""
    return lambda p: (1.0 / np.sqrt(p.astype(np.float64)) * (1.0 + rel)).astype(np.float32)


MUFU_REL = 2.0 ** -22.9


def test_float32_slope_tail_stays_inside_the_bound():
    """atan_sqrt_deg from the header's coefficients, with an exact reciprocal square root and with one off
    by the approximate instruction's worst relative error either way, is within 8 ulp32 + 1e-8 degrees of
    degrees(atan(sqrt(A^2 + B^2))) for A^2 + B^2 from 1e-14 to 1e8: what the GPU tests allow."""
    m2 = np.concatenate([np.geomspace(1e-14, 1e8, 400001),
                         np.tan(np.radians(np.linspace(1e-3, 89.99, 200001))) ** 2])
    tr = np.degrees(np.arctan(np.sqrt(m2)))
    worst = 0.0
    for rel in (0.0, MUFU_REL, -MUFU_REL):
        k = _tail_slope(m2, _rsqrt(rel)).astype(np.float64)
        e = np.abs(k - tr)
        assert (e <= 8 * ulp32(tr) + 1e-8).all(), (rel, (e / ulp32(tr)).max())
        worst = max(worst, float((e / ulp32(tr))[tr > 1e-5].max()))
    assert worst < 8.0, worst
    # neighbouring float32 inputs: the outputs step by at most two ulps (the bound between two float64
    # forms of the same plane, in the broadcast and antimeridian tests)
    p = np.tan(np.radians(np.linspace(1e-3, 89.9, 400001))).astype(np.float32) ** 2
    a = _tail_slope(p, _rsqrt(0.0)).astype(np.float64)
    b = _tail_slope(np.nextafter(p, np.float32(np.inf)), _rsqrt(0.0)).astype(np.float64)
    assert (np.abs(b - a) <= 2 * ulp32(a)).all()


def test_float32_compass_tail_stays_inside_the_bound():
    """compass_deg(-A, -B) as test_kernel_algebra states it, over a dense fan of directions (the axes
    exactly, both sides of each axis and of each octant boundary) and magnitudes 1e-7 .. 1e4, is within
    8 ulp32(max(aspect, 1)) of atan2(-A, -B) folded to [0, 360) in float64."""
    coeffs = [np.float32(x) for x in _atan_coeffs()]
    ang = np.concatenate([np.linspace(0.0, 360.0, 2881)[:-1],
                          np.repeat(np.arange(0.0, 360.0, 45.0), 4) + np.tile([-1e-4, -1e-6, 1e-6, 1e-4], 8)])
    worst = 0.0
    for mag in (3e-7, 1e-3, 1.0, 1e4):
        for t in np.radians(ang):
            A, B = -mag * np.sin(t), -mag * np.cos(t)
            if abs(A) < 1e-12 * mag:
                A = 0.0
            if abs(B) < 1e-12 * mag:
                B = 0.0
            ref = np.degrees(np.arctan2(-A, -B)) % 360.0
            for rel in (0.0, MUFU_REL, -MUFU_REL):
                # rcp.approx's error enters as the ratio t's relative error: scale the smaller magnitude
                u, v = np.float32(-A), np.float32(-B)
                if abs(u) < abs(v):
                    u = np.float32(np.float64(u) * (1 + rel))
                else:
                    v = np.float32(np.float64(v) * (1 + rel))
                got = float(_compass(u, v, coeffs))
                d = abs(got - ref)
                d = min(d, 360.0 - d)
                sc = ulp32(max(ref, 1.0))
                assert d <= 8 * sc + 1e-8, (mag, np.degrees(t), rel, got, ref)
                worst = max(worst, d / sc)
    assert worst < 8.0, worst


# ------------------------------------------------------------------------------------------- GPU
try:
    import torch
except ImportError:             # the CPU tests above need no torch
    torch = None


@pytest.fixture(scope="module", autouse=True)
def _report_the_largest_error():
    """Prints the largest kernel error over the module's cases (seen with -s)."""
    yield
    for key, (u, deg) in sorted(WORST.items()):
        print("\ngeodesic: largest kernel error over the suite, %s: %.2f ulp32 (T >= 1e-4 deg), %.3g deg" % (key, u, deg))


@pytest.fixture(scope="module")
def xb():
    import xrspatial_b200
    assert torch.cuda.is_available(), "these tests need a CUDA device"
    return xrspatial_b200


def dev(a, device="cuda"):
    return torch.from_numpy(np.ascontiguousarray(a)).to(device)


def da(xb, data, lat, lon):
    if np.ndim(lat) == 2:
        return xb.DataArray(data, dims=("lat", "lon"), coords={"latitude": lat, "longitude": lon})
    return xb.DataArray(data, dims=("lat", "lon"), coords={"lat": lat, "lon": lon})


def host(x):
    d = x.data
    return d.cpu().numpy() if hasattr(d, "cpu") else np.asarray(d)


def run(xb, data, lat, lon, aspect=False, z_unit="meter"):
    g = da(xb, data, lat, lon)
    f = xb.aspect if aspect else xb.slope
    return host(f(g, method="geodesic", z_unit=z_unit))


def both(xb, c, what, data=None, z_unit="meter", ex=None):
    """slope and aspect of case `c` through the public API, each against T and the oracle."""
    data = dev(c["z"]) if data is None else data
    ex = c["ex"] if ex is None else ex
    s = run(xb, data, c["lat"], c["lon"], z_unit=z_unit)
    a = run(xb, data, c["lat"], c["lon"], aspect=True, z_unit=z_unit)
    check(s, ex, what)
    check(a, ex, what, aspect=True)
    return s, a


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("dt", [np.float64, np.float32], ids=["f64", "f32"])
def test_cases_meet_the_bound(xb, cases, name, dt):
    """Every fixture in float64 and float32 cells (1-D fixtures run geodesic_kernel<T, false>, 2-D ones
    geodesic_kernel<T, true>), slope and aspect within the bound of T."""
    both(xb, cases[name, dt], "%s %s" % (name, dt.__name__))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["46N_descending_1s", "irregular_1s", "antimeridian_wrapped", "spacing_30s"])
@pytest.mark.parametrize("dt", [np.float64, np.float32], ids=["f64", "f32"])
def test_broadcast_2d_coordinates_match_the_1d_call(xb, cases, name, dt):
    """2-D coordinates that are the broadcast of a 1-D grid take the ECEF path; the 1-D call takes the folded
    tables.  Both meet T, and they differ by at most two float32 ulps: where the two float64 forms of
    A^2 + B^2 round to neighbouring float32 values, the float32 tail can step by two ulps (see the tail
    test)."""
    c = cases[name, dt]
    la2, lo2 = _b2(c["lat"], c["lon"], c["z"].shape)
    data = dev(c["z"])
    s2, a2 = both(xb, dict(c, lat=la2, lon=lo2), "%s 2-D broadcast %s" % (name, dt.__name__), data=data)
    s1, a1 = run(xb, data, c["lat"], c["lon"]), run(xb, data, c["lat"], c["lon"], aspect=True)
    m = np.isfinite(s1)
    d = np.abs(s1[m].astype(np.float64) - s2[m])
    assert (d <= 2 * ulp32(np.maximum(s1[m], s2[m]))).all(), d.max()
    m = np.isfinite(a1) & (a1 != -1)
    d = np.abs(a1[m].astype(np.float64) - a2[m])
    d = np.minimum(d, 360.0 - d)
    assert (d <= 2 * ulp32(np.maximum(np.maximum(a1[m], a2[m]), 1.0))).all(), d.max()


@pytest.mark.gpu
def test_antimeridian_forms_agree(xb, cases):
    """179.99 .. -179.99 (wrapped, non-monotonic) and 179.99 .. 180.01 describe the same cells: within two
    float32 ulps of each other, the tail's step between neighbouring inputs."""
    for dt in (np.float64, np.float32):
        cw, c0 = cases["antimeridian_wrapped", dt], cases["antimeridian_0_360", dt]
        assert (np.diff(cw["lon"]) < 0).any() and (np.diff(c0["lon"]) > 0).all()
        np.testing.assert_array_equal(cw["z"], c0["z"])
        for aspect in (False, True):
            w = run(xb, dev(cw["z"]), cw["lat"], cw["lon"], aspect=aspect)
            z = run(xb, dev(c0["z"]), c0["lat"], c0["lon"], aspect=aspect)
            np.testing.assert_array_equal(np.isnan(w), np.isnan(z))
            m = np.isfinite(w) & (w != -1)
            d = np.abs(w[m].astype(np.float64) - z[m])
            d = np.minimum(d, 360.0 - d) if aspect else d
            assert (d <= 2 * ulp32(np.maximum(np.maximum(w[m], z[m]), 1.0 if aspect else 0.0))).all(), d.max()


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.int16, np.int32])
def test_integer_elevation(xb, dt):
    """Integer cells are computed as their float64 values (slope.py:169): the float64 call's bits, and T."""
    c = regular(axis(46.0, -3 * S1, 40), axis(7.0, 3 * S1, 52), seed=12)
    z = np.round(c["z"]).astype(dt)
    ex = expect(z, c["lat"], c["lon"])
    s, a = both(xb, dict(c, z=z), "integer " + np.dtype(dt).name, ex=ex)
    np.testing.assert_array_equal(bits(s), bits(run(xb, dev(z.astype(np.float64)), c["lat"], c["lon"])))
    np.testing.assert_array_equal(bits(a), bits(run(xb, dev(z.astype(np.float64)), c["lat"], c["lon"], aspect=True)))


@pytest.mark.gpu
@pytest.mark.parametrize("unit,factor", [("meter", 1.0), ("foot", 0.3048), ("km", 1000.0), ("mile", 1609.344)])
@pytest.mark.parametrize("dt", [np.float64, np.float32], ids=["f64", "f32"])
def test_z_units(xb, unit, factor, dt):
    """Elevation in feet, kilometres and miles is scaled by the z factor before the frame change."""
    c = regular(axis(46.0, -S1, 40), axis(7.0, S1, 52), seed=13)
    z = (c["z"] / factor).astype(dt)
    both(xb, dict(c, z=z), "z_unit %s %s" % (unit, dt.__name__), z_unit=unit, ex=expect(z, c["lat"], c["lon"], factor))


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float64, np.float32], ids=["f64", "f32"])
def test_nan_elevation_blanks_exactly_its_neighbourhood(xb, dt):
    """One NaN cell inside the raster, on an edge row, on an edge column and in a corner: NaN on exactly its
    3 x 3 neighbourhood and the raster's ring; every other cell meets the bound."""
    c = regular(axis(46.0, -S1, 40), axis(7.0, S1, 52), seed=14)
    H, W = c["z"].shape
    for (y, x) in ((17, 23), (0, 30), (25, W - 1), (H - 1, 0)):
        z = c["z"].astype(dt)
        z[y, x] = np.nan
        want = np.zeros((H, W), bool)
        want[[0, -1], :] = want[:, [0, -1]] = True
        want[max(0, y - 1):y + 2, max(0, x - 1):x + 2] = True
        s, a = both(xb, dict(c, z=z), "NaN at %d,%d %s" % (y, x, dt.__name__), ex=expect(z, c["lat"], c["lon"]))
        np.testing.assert_array_equal(np.isnan(s), want)
        np.testing.assert_array_equal(np.isnan(a), want)


@pytest.mark.gpu
def test_nan_coordinates_blank_the_cells_that_use_them(xb):
    """A NaN latitude row, a NaN longitude column (1-D) and a NaN 2-D coordinate cell give NaN where the
    oracle does, and the bound elsewhere."""
    c = regular(axis(46.0, -S1, 40), axis(7.0, S1, 52), seed=15)
    lat, lon = c["lat"].copy(), c["lon"].copy()
    lat[11] = np.nan
    lon[0] = np.nan
    lon[30] = np.nan
    s, a = both(xb, dict(c, lat=lat, lon=lon), "NaN lat row / lon columns", ex=expect(c["z"], lat, lon))
    assert np.isnan(s[10:13]).all() and np.isnan(s[:, 29:32]).all() and np.isnan(s[:, 1]).all()
    assert np.isfinite(s[14:20, 3:28]).all()
    k = curvilinear("rotated", seed=3)
    la2, lo2 = k["lat"].copy(), k["lon"].copy()
    la2[20, 20] = np.nan
    lo2[5, 40] = np.nan
    s, _ = both(xb, dict(k, lat=la2, lon=lo2), "NaN 2-D coordinates", ex=expect(k["z"], la2, lo2))
    assert np.isnan(s[19:22, 19:22]).all() and np.isnan(s[4:7, 39:42]).all()


def _plane(lat, lon, grade, bearing):
    """Elevation of a plane falling at `grade` (rise over run) toward compass `bearing`, in local metres."""
    la2, lo2 = _b2(lat, lon, (len(lat), len(lon)))
    e2 = 1.0 - float(B2 / A2)
    w = 1.0 - e2 * np.sin(np.radians(la2)) ** 2                 # meridian and prime-vertical radii of WGS-84
    y = np.radians(la2 - la2[0, 0]) * 6378137.0 * (1.0 - e2) / w ** 1.5
    x = np.radians(lo2 - lo2[0, 0]) * 6378137.0 / np.sqrt(w) * np.cos(np.radians(la2))
    b = np.radians(bearing)
    return 500.0 - grade * (x * np.sin(b) + y * np.cos(b))


@pytest.mark.gpu
def test_flat_surface_and_the_flat_threshold(xb):
    """A flat surface gives slope 0 (within the bound) and aspect -1; float64 planes with |(A, B)| 3 x above
    and 3 x below 1e-7 give the oracle's flat mask."""
    lat, lon = axis(46.0, -S1, 24), axis(7.0, S1, 30)
    c = dict(z=np.full((24, 30), 812.5), lat=lat, lon=lon)
    c["ex"] = expect(c["z"], lat, lon)
    s, a = both(xb, c, "flat")
    assert (s[1:-1, 1:-1] < 1e-6).all() and (a[1:-1, 1:-1] == -1).all()
    lat, lon = axis(46.0, -300 * S1, 24), axis(7.0, 300 * S1, 30)    # 5' cells: float64 resolves 3e-7
    for g, flat in ((3e-7, False), (3e-8, True)):
        z = _plane(lat, lon, g, 37.0)
        ex = expect(z, lat, lon)
        mag = ex["mag"][1:-1, 1:-1].astype(np.float64)
        assert ((mag < 1e-7 / 3) if flat else (mag > 3e-7 * 0.9)).all(), (mag.min(), mag.max())
        _, a = both(xb, dict(z=z, lat=lat, lon=lon), "plane |(A, B)| = %g" % g, ex=ex)
        assert ((a[1:-1, 1:-1] == -1) == flat).all()


@pytest.mark.gpu
@pytest.mark.parametrize("lat0", [0.0, 60.0])
def test_sixteen_downslope_directions(xb, lat0):
    """Planes falling toward 16 bearings, N / E / S / W exactly among them: aspect within the bound of T and
    within 0.05 degrees of the plane's bearing."""
    lat, lon = axis(lat0 + 12 * S1, -S1, 24), axis(30.0, S1, 30)
    for k in range(16):
        bearing = 22.5 * k
        z = _plane(lat, lon, 0.3, bearing)
        _, a = both(xb, dict(z=z, lat=lat, lon=lon), "bearing %.1f at %g" % (bearing, lat0),
                    ex=expect(z, lat, lon))
        d = np.abs(a[1:-1, 1:-1].astype(np.float64) - bearing)
        assert (np.minimum(d, 360.0 - d) < 0.05).all(), (bearing, d.max())


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(1, 7), (2, 7), (3, 7), (7, 1), (7, 2), (7, 3), (1, 1), (2, 2), (3, 3)])
def test_small_shapes(xb, shape):
    """Below 3 rows or columns every cell is on the ring: all NaN.  3 x 3 has exactly one cell."""
    H, W = shape
    c = regular(axis(46.0, -S1, H), axis(7.0, S1, W), seed=16)
    for dt in (np.float64, np.float32):
        z = c["z"].astype(dt)
        both(xb, dict(c, z=z), "shape %dx%d %s" % (H, W, dt.__name__), ex=expect(z, c["lat"], c["lon"]))
        k = curvilinear("rotated", H=H, W=W)
        both(xb, dict(k, z=k["z"].astype(dt)), "shape %dx%d 2-D %s" % (H, W, dt.__name__),
             ex=expect(k["z"].astype(dt), k["lat"], k["lon"]))


def _pass_cells():
    """Cells one launch covers before its grid-stride loop wraps: sm_count * 8 CTAs of 256 threads."""
    return torch.cuda.get_device_properties(0).multi_processor_count * 8 * 256


@pytest.mark.gpu
@pytest.mark.parametrize("where", ["below_one_pass", "above_one_pass", "over_two_passes"])
def test_launch_sizes(xb, where):
    """H * W just below and just above one pass of the grid-stride loop, and beyond two passes."""
    cap, W = _pass_cells(), 509
    H = {"below_one_pass": cap // W, "above_one_pass": cap // W + 1, "over_two_passes": 2 * cap // W + 3}[where]
    assert (H * W <= cap) == (where == "below_one_pass")
    c = regular(axis(46.0, -S1, H), axis(7.0, S1, W), seed=17)
    c["ex"] = expect(c["z"], c["lat"], c["lon"])
    both(xb, c, "launch %s %dx%d" % (where, H, W))
    z32 = c["z"].astype(np.float32)
    check(run(xb, dev(z32), c["lat"], c["lon"]), expect(z32, c["lat"], c["lon"]), "launch %s f32" % where)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(100000, 3), (3, 200000)])
def test_long_thin_rasters(xb, shape):
    """geo_tables_kernel covers max(H, W) rows and columns in one grid."""
    H, W = shape
    lat = axis(46.0, -S1, H) if H > 3 else axis(46.0, -30 * S1, H)
    lon = axis(7.0, S1, W) if W > 3 else axis(7.0, 30 * S1, W)
    c = regular(lat, lon, seed=18)
    c["ex"] = expect(c["z"], lat, lon)
    both(xb, c, "long thin %dx%d" % shape)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float64, np.float32], ids=["f64", "f32"])
def test_views_streams_and_host_input_are_bit_identical(xb, cases, dt):
    """A column slice (pitch > W, base off 16-byte alignment), a row-offset view, a call on a side stream,
    numpy input (1-D and 2-D coordinates, numpy output) and a second device give the contiguous call's
    bits."""
    c = cases["irregular_1s", dt]
    z, lat, lon = c["z"], c["lat"], c["lon"]
    H, W = z.shape
    la2, lo2 = _b2(lat, lon, z.shape)
    for aspect in (False, True):
        ref = run(xb, dev(z), lat, lon, aspect=aspect)
        ref2 = run(xb, dev(z), la2, lo2, aspect=aspect)
        big = np.full((H + 9, W + 14), 9.0e3, dtype=dt)    # W even: an odd element offset, 8 or 4 mod 16 bytes
        big[5:5 + H, 3:3 + W] = z
        t = dev(big)
        col = t[5:5 + H, 3:3 + W]
        assert col.stride(0) == W + 14 and (col.data_ptr() % 16) != 0
        np.testing.assert_array_equal(bits(run(xb, col, lat, lon, aspect=aspect)), bits(ref))
        np.testing.assert_array_equal(bits(run(xb, col, la2, lo2, aspect=aspect)), bits(ref2))
        rows = dev(np.concatenate([np.full((7, W), -3.0e3, dt), z, np.full((2, W), 7.0e3, dt)]))[7:7 + H]
        np.testing.assert_array_equal(bits(run(xb, rows, lat, lon, aspect=aspect)), bits(ref))
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            d = dev(z)
            out = (xb.aspect if aspect else xb.slope)(da(xb, d, lat, lon), method="geodesic").data
        side.synchronize()
        np.testing.assert_array_equal(bits(out.cpu().numpy()), bits(ref))
        for la, lo, want in ((lat, lon, ref), (la2, lo2, ref2)):
            h = (xb.aspect if aspect else xb.slope)(da(xb, z, la, lo), method="geodesic").data
            assert isinstance(h, np.ndarray)
            np.testing.assert_array_equal(bits(h), bits(want))
        if torch.cuda.device_count() > 1:
            d1 = dev(z, "cuda:1")
            out = (xb.aspect if aspect else xb.slope)(da(xb, d1, lat, lon), method="geodesic").data
            assert out.device == d1.device
            np.testing.assert_array_equal(bits(out.cpu().numpy()), bits(ref))


@pytest.mark.gpu
def test_4096_square_one_arcsecond_grid_against_the_oracle(xb):
    """A 4096 x 4096 1-arcsecond float64 grid: within 8 ulp32(oracle) + 1e-8 degrees of the oracle."""
    n = 4096
    lat, lon = axis(46.0, -S1, n), axis(7.0, S1, n)
    z = surface(*_b2(lat, lon, (n, n)), seed=19)
    la2, lo2 = _b2(lat, lon, z.shape)
    ref = o.geodesic(z, la2, lo2, nthreads=o.max_threads())
    got = run(xb, dev(z), lat, lon)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
    m = np.isfinite(ref)
    d = np.abs(got[m].astype(np.float64) - ref[m])
    u = ulp32(ref[m])
    assert (d <= 8 * u + 1e-8).all(), (d / u).max()
    print("geodesic 4096x4096 vs oracle: max %.2f ulp32  %.3g deg" % ((d / u).max(), d.max()))

"""Pins the CPU oracle (oracle/xrs_oracle.c, oracle/oracle.py) against

(a) the known-answer arrays of the reference's own test-suite (tests/golden/known_answers.npz,
    extracted from the reference's xrspatial/tests by oracle/make_golden.py) and
(b) outputs of the unmodified reference kernels on seeded inputs
    (tests/golden/reference_outputs.npz).

CPU only; runs in seconds.
"""
import numpy as np
import pytest

import oracle as o

DEMS = ["smooth", "water", "nans", "integer", "rough", "tiny", "rand_2x4", "rand_10x15"]
STATS = ["mean", "max", "min", "range", "std", "var", "sum"]


def same_nan(a, b):
    np.testing.assert_array_equal(np.isnan(a), np.isnan(b))


# ----------------------------------------------------------------- (a) known answers
def test_slope_qgis(known):
    # test_slope.py:22-49 (res=(1,1), interior compared at rtol 1e-5)
    out = o.slope(known["conftest.elevation_raster"], 1, 1)
    np.testing.assert_allclose(out[1:-1, 1:-1], known["slope.qgis_slope"][1:-1, 1:-1],
                               rtol=1e-5, equal_nan=True)
    assert out.dtype == np.float32
    assert np.isnan(out[0]).all() and np.isnan(out[-1]).all()
    assert np.isnan(out[:, 0]).all() and np.isnan(out[:, -1]).all()


def test_slope_docstring():
    # slope.py:317-331
    data = np.array([[0, 0, 0, 0, 0], [0, 0, 0, -1, 2], [0, 0, 0, 0, 1], [0, 0, 0, 5, 0]])
    exp = np.array([[0., 14.036243, 32.512516], [0., 42.031113, 53.395725]], dtype=np.float32)
    np.testing.assert_allclose(o.slope(data, 1, 1)[1:3, 1:4], exp, rtol=1e-6)


def test_aspect_qgis(known):
    # test_aspect.py:19-47
    out = o.aspect(known["conftest.elevation_raster"])
    np.testing.assert_allclose(out[1:-1, 1:-1], known["aspect.qgis_aspect"][1:-1, 1:-1],
                               rtol=1e-5, equal_nan=True)


@pytest.mark.parametrize("surf", ["convex_surface", "concave_surface"])
def test_curvature_known(known, surf):
    # test_curvature.py:26-84 (res (1,1) -> cellsize 1)
    out = o.curvature(known["curvature.%s.data" % surf], 1)
    np.testing.assert_allclose(out, known["curvature.%s.expected" % surf], equal_nan=True)


def test_curvature_flat():
    out = o.curvature(np.zeros((5, 7)), 1)
    assert (out[1:-1, 1:-1] == 0).all() and np.signbit(out[1:-1, 1:-1]).all()  # -0.0


def test_hillshade_docstring():
    # hillshade.py:153-170 (the only numeric pin the reference has for hillshade)
    data = np.array([[0., 0., 0., 0., 0.], [0., 1., 0., 2., 0.], [0., 0., 3., 0., 0.],
                     [0., 0., 0., 0., 0.], [0., 0., 0., 0., 0.]])
    exp = np.array([[0.71130913, 0.44167341, 0.71130913],
                    [0.95550163, 0.71130913, 0.52478473],
                    [0.71130913, 0.88382559, 0.71130913]])
    np.testing.assert_allclose(o.hillshade(data)[1:4, 1:4], exp, rtol=1e-6)


def test_convolution_known(known):
    # test_focal.py:113-225
    data = known["focal.convolve_2d_data"]
    for k, e in (("focal.kernel_circle_1_1_1", "focal.convolution_kernel_circle_1_1_1"),
                 ("focal.kernel_annulus_2_2_2_1", "focal.convolution_kernel_annulus_2_2_1"),
                 ("focal.convolution_custom_kernel.kernel", "focal.convolution_custom_kernel.expected")):
        np.testing.assert_allclose(o.convolve_2d(data, known[k]), known[e], equal_nan=True)


def test_focal_stats_known(known):
    # test_focal.py:353-404
    data, kernel = known["focal.data_focal_stats.data"], known["focal.data_focal_stats.kernel"]
    exp = known["focal.data_focal_stats.expected"]
    for i, s in enumerate(STATS):
        np.testing.assert_allclose(o.focal_apply(data, kernel, s), exp[i], rtol=1e-6, err_msg=s)


def test_focal_mean_docstring():
    # focal.py:195-209
    data = np.array([[0., 0., 0., 0., 0.], [0., 1., 1., 1., 0.], [0., 1., 1., 1., 0.],
                     [0., 1., 1., 1., 0.], [0., 0., 0., 0., 0.]])
    out = o.focal_mean(data)
    assert out.dtype == np.float64
    np.testing.assert_allclose(out[0, :3], [0.25, 0.33333333, 0.5], rtol=1e-7)
    np.testing.assert_allclose(out[2, 2], 1.0)


MS_QGIS = {
    "ndvi": ("normalized_ratio", ("nir", "red")), "nbr": ("normalized_ratio", ("nir", "swir2")),
    "nbr2": ("normalized_ratio", ("swir1", "swir2")), "ndmi": ("normalized_ratio", ("nir", "swir1")),
    "savi": ("savi", ("nir", "red")), "evi": ("evi", ("nir", "red", "blue")),
    "arvi": ("arvi", ("nir", "red", "blue")), "gci": ("gci", ("nir", "green")),
    "sipi": ("sipi", ("nir", "red", "blue")), "ebbi": ("ebbi", ("red", "swir1", "tir")),
}


@pytest.mark.parametrize("name", sorted(MS_QGIS))
def test_multispectral_qgis(known, name):
    # test_multispectral.py:12-283, compared like general_output_checks (rtol 1e-6 default
    # there is loosened by the QGIS tables' 7-8 significant digits -> rtol 1e-5)
    fn, bands = MS_QGIS[name]
    out = getattr(o, fn)(*[known["multispectral.%s_data" % b] for b in bands])
    np.testing.assert_allclose(out, known["multispectral.qgis_" + name], rtol=1e-5, atol=1e-7,
                               equal_nan=True)


def test_multispectral_uint(known):
    # test_multispectral.py:285-338
    g = lambda n, i: known["multispectral.uint_%s.%d" % (n, i)]  # noqa: E731
    np.testing.assert_allclose(o.normalized_ratio(g("normalized_ratio", 0), g("normalized_ratio", 1)),
                               g("normalized_ratio", 2), rtol=1e-6)
    np.testing.assert_allclose(o.arvi(g("arvi", 0), g("arvi", 1), g("arvi", 2)), g("arvi", 3), rtol=1e-6)
    np.testing.assert_allclose(o.evi(g("evi", 0), g("evi", 1), g("evi", 2)), g("evi", 3), rtol=1e-6)
    np.testing.assert_allclose(o.savi(g("savi", 0), g("savi", 1)), g("savi", 2), rtol=1e-6)
    np.testing.assert_allclose(o.sipi(g("sipi", 0), g("sipi", 1), g("sipi", 2)), g("sipi", 3), rtol=1e-6)
    np.testing.assert_allclose(o.ebbi(g("ebbi", 0), g("ebbi", 1), g("ebbi", 2)), g("ebbi", 3), rtol=1e-6)


def test_zonal_known(known):
    # test_zonal.py:30-75, 131-146, 339-385, 593-602
    zones, values = known["zonal.data_zones"], known["zonal.data_values_2d"]
    res = o.zonal_stats(zones, values, stats_funcs=["mean", "max", "min", "sum", "std", "var", "count", "majority"])
    for k in ("zone", "mean", "max", "min", "sum", "std", "var", "count", "majority"):
        np.testing.assert_allclose(res[k], known["zonal.result_default_stats." + k], rtol=1e-5, atol=1e-7)
    res = o.zonal_stats(zones, values, zone_ids=list(known["zonal.result_zone_ids_stats.zone_ids"]))
    for k in ("zone", "mean", "max", "min", "sum", "std", "var", "count"):
        np.testing.assert_allclose(res[k], known["zonal.result_zone_ids_stats." + k], rtol=1e-5, atol=1e-7)
    res = o.zonal_stats(known["conftest.raster"], known["conftest.elevation_raster_no_nans"],
                        stats_funcs=["mean", "max", "min", "sum", "count"])
    for k in ("zone", "mean", "max", "min", "sum", "count"):
        np.testing.assert_allclose(res[k], known["zonal.qgis_zonal_stats." + k], rtol=1e-5, atol=1e-5)


# --------------------------------------------------- (b) outputs of the reference itself
@pytest.mark.parametrize("case", DEMS)
def test_surface_vs_reference(refout, case):
    z = refout["dem." + case]
    # f64 arithmetic restated exactly -> identical after rounding to f32
    np.testing.assert_array_equal(o.slope(z, 30.0, 30.0), refout["slope." + case])
    np.testing.assert_array_equal(o.slope(z, 10.0, 25.5), refout["slope_aniso." + case])
    np.testing.assert_array_equal(o.aspect(z), refout["aspect." + case])
    np.testing.assert_array_equal(o.curvature(z, 30.0), refout["curvature." + case])
    # NumPy's SIMD float32 transcendentals vs libm: a few f32 ulp on values in [0, 1]
    np.testing.assert_allclose(o.hillshade(z, 225, 25), refout["hillshade." + case],
                               rtol=0, atol=5e-7, equal_nan=True)
    np.testing.assert_allclose(o.hillshade(z, 315, 45), refout["hillshade_az315_alt45." + case],
                               rtol=0, atol=5e-7, equal_nan=True)


@pytest.mark.parametrize("case", DEMS)
def test_focal_mean_vs_reference(refout, case):
    z = refout["dem." + case]
    np.testing.assert_array_equal(o.focal_mean(z), refout["focal_mean." + case])
    np.testing.assert_array_equal(o.focal_mean(z, passes=3), refout["focal_mean_p3." + case])
    np.testing.assert_array_equal(o.focal_mean(z, excludes=(np.nan, 0.0)), refout["focal_mean_ex." + case])


@pytest.mark.parametrize("kn", ["box3", "box9", "mixed5", "mixed3x7", "mixed25", "int3"])
def test_convolve_vs_reference(refout, kn):
    k = refout["conv.kernel." + kn]
    np.testing.assert_array_equal(o.convolve_2d(refout["conv.dem"], k), refout["conv.out." + kn])
    np.testing.assert_array_equal(o.convolve_2d(refout["conv.dem_nan"], k), refout["conv.out_nan." + kn])


@pytest.mark.parametrize("mn", ["circle3", "full3", "annulus5", "rect3x5", "weights3"])
def test_focal_apply_vs_reference(refout, mn):
    for s in STATS:
        np.testing.assert_array_equal(o.focal_apply(refout["apply.dem"], refout["apply.mask." + mn], s),
                                      refout["apply.out.%s.%s" % (mn, s)], err_msg=s)


@pytest.mark.parametrize("kh,kw", [(5, 5), (25, 25), (3, 7), (9, 3)])
def test_focal_apply_mean_over_all_ones_windows_vs_reference(refout, kh, kw):
    """focal.apply(raster, np.ones((kh, kw))) -- the shapes of the reference's FocalApply benchmark -- run through
    the unmodified reference (`_apply_numpy` + `_calc_mean`) on a raster with NaNs, an all-NaN patch, +-inf and a
    FLT_MAX-style sentinel: the oracle the GPU's NaN-skipping running box is checked against gives the same bits."""
    ref = refout["apply_ones.mean.%dx%d" % (kh, kw)]
    np.testing.assert_array_equal(o.focal_apply(refout["apply_ones.dem"], np.ones((kh, kw)), "mean"), ref)
    assert np.isinf(ref).any() and (np.isnan(ref).any() or kh * kw > 120)     # the 10 x 12 all-NaN patch is smaller than 25 x 25


def test_multispectral_vs_reference(refout):
    r = refout
    np.testing.assert_array_equal(o.normalized_ratio(r["ms.nir"], r["ms.red"]), r["ms.ndvi"])
    np.testing.assert_array_equal(o.savi(r["ms.nir"], r["ms.red"], 1.0), r["ms.savi"])
    np.testing.assert_array_equal(o.savi(r["ms.nir"], r["ms.red"], 0.5), r["ms.savi_L05"])
    np.testing.assert_array_equal(o.evi(r["ms.nir"], r["ms.red"], r["ms.blue"]), r["ms.evi"])
    np.testing.assert_array_equal(o.arvi(r["ms.nir"], r["ms.red"], r["ms.blue"]), r["ms.arvi"])
    np.testing.assert_array_equal(o.gci(r["ms.nir"], r["ms.green"]), r["ms.gci"])
    np.testing.assert_array_equal(o.sipi(r["ms.nir"], r["ms.red"], r["ms.blue"]), r["ms.sipi"])
    np.testing.assert_array_equal(o.ebbi(r["ms.red"], r["ms.swir"], r["ms.tir"]), r["ms.ebbi"])


def test_zonal_vs_reference(refout):
    r = refout
    cols = ["zone", "mean", "max", "min", "sum", "std", "var", "count"]
    res = o.zonal_stats(r["zonal.zones_i32"], r["zonal.values_f32"],
                        stats_funcs=cols[1:] + ["majority"])
    for c in cols + ["majority"]:
        np.testing.assert_array_equal(res[c], r["zonal.f32_i32." + c], err_msg=c)
    res = o.zonal_stats(r["zonal.zones_i32"], r["zonal.values_f32"], zone_ids=[3, 7, 100, 999],
                        nodata_values=0.0)
    for c in cols:
        np.testing.assert_array_equal(res[c], r["zonal.f32_i32_ids_nodata." + c], err_msg=c)
    res = o.zonal_stats(r["zonal.zones_f64"], r["zonal.values_f64"])
    for c in cols:
        np.testing.assert_array_equal(res[c], r["zonal.f64_f64." + c], err_msg=c)


def test_threads_do_not_change_results(refout):
    z = refout["dem.smooth"]
    np.testing.assert_array_equal(o.slope(z, 30, 30, nthreads=4), o.slope(z, 30, 30))
    np.testing.assert_array_equal(o.focal_mean(z, nthreads=4), o.focal_mean(z))


def test_hotspots_vs_reference(refout):
    r = refout
    np.testing.assert_array_equal(o.hotspots(r["hotspots.dem"], r["hotspots.kernel"]), r["hotspots.out"])
    np.testing.assert_array_equal(o.hotspots(r["hotspots.dem"], np.ones((5, 5))), r["hotspots.out_5x5"])
    assert set(np.unique(r["hotspots.out"])) - {0} != set()      # the fixture really has hot / cold cells


def test_hotspots_classification_at_the_thresholds(refout):
    """float32 z within +-2048 ulps of +-every threshold, signed zeros, NaN, +-inf: the reference compares
    in float64, so z = +-1.96f (which is above 1.96) is +-95, not +-90."""
    z, ref = refout["hotspots.classify.z"], refout["hotspots.classify.out"]
    got = o.hotspots_classify(z)
    assert got.dtype == np.int8
    np.testing.assert_array_equal(got, ref)
    assert ref[z == np.float32(1.96)] == 95 and ref[z == -np.float32(1.96)] == -95


def test_crosstab_vs_reference(refout):
    r = refout
    for agg in ("count", "percentage"):
        res = o.crosstab(r["crosstab.zones"], r["crosstab.values"], agg=agg)
        cols = [c for c in res if not isinstance(c, str)]
        np.testing.assert_array_equal(np.asarray(cols, dtype=np.float64), r["crosstab.%s.columns" % agg])
        table = np.column_stack([res["zone"]] + [res[c] for c in cols]).astype(np.float64)
        np.testing.assert_allclose(table, r["crosstab.%s.table" % agg], rtol=1e-6, equal_nan=True)
    res = o.crosstab(r["crosstab.zones"], r["crosstab.values"], zone_ids=[1, 3, 9], cat_ids=[11.0, 13.0],
                     nodata_values=12.0)
    table = np.column_stack([res["zone"], res[11.0], res[13.0]]).astype(np.float64)
    np.testing.assert_array_equal(table, r["crosstab.sub.table"])


def test_geodesic_vs_reference(refout):
    r = refout
    z = r["geodesic.dem"]
    lat2 = np.broadcast_to(r["geodesic.lat"][:, None], z.shape)
    lon2 = np.broadcast_to(r["geodesic.lon"][None, :], z.shape)
    # libm vs Numba's sin/cos may differ in the last f64 bit -> compare the f32 outputs closely
    np.testing.assert_allclose(o.geodesic(z, lat2, lon2), r["geodesic.slope"], rtol=1e-6, atol=1e-7, equal_nan=True)
    np.testing.assert_allclose(o.geodesic(z, lat2, lon2, z_factor=0.3048), r["geodesic.slope_ft"], rtol=1e-6,
                               atol=1e-7, equal_nan=True)
    np.testing.assert_allclose(o.geodesic(z, lat2, lon2, aspect=True), r["geodesic.aspect"], rtol=1e-6, atol=1e-4,
                               equal_nan=True)
    np.testing.assert_allclose(o.geodesic(z, r["geodesic.lat2d"], r["geodesic.lon2d"]), r["geodesic.slope_2d"],
                               rtol=1e-6, atol=1e-7, equal_nan=True)
    np.testing.assert_allclose(o.geodesic(z, r["geodesic.lat2d"], r["geodesic.lon2d"], aspect=True),
                               r["geodesic.aspect_2d"], rtol=1e-6, atol=1e-4, equal_nan=True)
    assert (r["geodesic.aspect"] == -1).any() and np.isnan(r["geodesic.slope"][1:-1, 1:-1]).any()


# ----------------------------------------------------------------- geodesic: the reference's own property tests
# tests/test_geodesic_slope.py:76-199 and tests/test_geodesic_aspect.py:81-190 hold no tables, only
# analytical expectations on small coarse grids (1 degree over 6 x 8 cells); the oracle must meet them.
def _geo_grid(elev, la0, la1, lo0=10.0, lo1=11.0):
    h, w = elev.shape
    lat, lon = np.linspace(la0, la1, h), np.linspace(lo0, lo1, w)
    return np.broadcast_to(lat[:, None], (h, w)).copy(), np.broadcast_to(lon[None, :], (h, w)).copy(), lat, lon


def _tilted(axis, sign, h=6, w=8, grade=100.0):
    ramp = np.linspace(0.0, 1.0, w if axis == "east" else h) * grade * sign
    return (np.broadcast_to(500.0 + ramp[None, :], (h, w)) if axis == "east"
            else np.broadcast_to(500.0 + ramp[:, None], (h, w))).copy()


@pytest.mark.parametrize("lat_center", [0.0, 30.0, 60.0, -45.0])
def test_geodesic_flat_surface_like_reference_tests(lat_center):
    flat = np.full((6, 8), 500.0)
    la, lo, _, _ = _geo_grid(flat, lat_center - 0.5, lat_center + 0.5)
    s = o.geodesic(flat, la, lo)
    assert np.isfinite(s[1:-1, 1:-1]).all()
    np.testing.assert_allclose(s[1:-1, 1:-1], 0.0, atol=0.1)             # test_geodesic_slope.py:76-89
    a = o.geodesic(flat, la, lo, aspect=True)
    np.testing.assert_allclose(a[1:-1, 1:-1], -1.0, atol=1e-4)           # test_geodesic_aspect.py:81-87
    for out in (s, a):                                                    # edges are NaN (:152-160 / :144-151)
        assert np.isnan(out[0]).all() and np.isnan(out[-1]).all() and np.isnan(out[:, 0]).all() and np.isnan(out[:, -1]).all()


def test_geodesic_tilted_surfaces_like_reference_tests():
    expect = {("east", 1): 270.0, ("north", 1): 180.0, ("north", -1): 0.0, ("east", -1): 90.0}
    for (axis, sign), asp in expect.items():
        z = _tilted(axis, sign)
        la, lo, _, _ = _geo_grid(z, 40.0, 41.0)
        s = o.geodesic(z, la, lo)[1:-1, 1:-1]
        assert np.isfinite(s).all() and (s > 0).all()                     # test_geodesic_slope.py:92-109
        a = float(o.geodesic(z, la, lo, aspect=True)[2, 4])               # test_geodesic_aspect.py:89-131
        d = abs(a - asp)
        assert min(d, 360.0 - d) < 5.0, (axis, sign, a)
    # latitude invariance (:112-137): the same grade per degree of longitude is ~2x steeper at 60N
    z = _tilted("east", 1, grade=50.0)
    s_eq = o.geodesic(z, *_geo_grid(z, -0.5, 0.5)[:2])[2, 4]
    s_60 = o.geodesic(z, *_geo_grid(z, 59.5, 60.5)[:2])[2, 4]
    assert s_eq > 0 and 1.5 < s_60 / s_eq < 2.5
    # near the pole (:162-173) and feet vs metres (:179-199)
    zp = _tilted("north", 1, h=6, w=6, grade=50.0)
    sp = o.geodesic(zp, *_geo_grid(zp, 88.0, 89.0)[:2])[1:-1, 1:-1]
    assert np.isfinite(sp).all() and (sp > 0).all()
    zm = _tilted("east", 1)
    la, lo, _, _ = _geo_grid(zm, 40.0, 41.0)
    np.testing.assert_allclose(o.geodesic(zm, la, lo)[1:-1, 1:-1],
                               o.geodesic(zm / 0.3048, la, lo, z_factor=0.3048)[1:-1, 1:-1], rtol=1e-4)
    # NaN in the neighbourhood (:140-150)
    zn = np.full((5, 5), 500.0)
    zn[2, 2] = np.nan
    sn = o.geodesic(zn, *_geo_grid(zn, 40.0, 41.0)[:2])
    assert np.isnan(sn[2, 2]) and np.isnan(sn[1, 1]) and np.isnan(sn[1, 2])
    # aspect range (:153-166)
    zr = np.random.default_rng(42).uniform(100, 1000, size=(10, 10))
    ar = o.geodesic(zr, *_geo_grid(zr, 40.0, 41.0)[:2], aspect=True)[1:-1, 1:-1]
    d = ar[np.isfinite(ar) & (ar != -1.0)]
    assert (d >= 0.0).all() and (d < 360.0).all()


def _geodesic_folded(z, lat, lon, zf=1.0, aspect=False):
    """NumPy statement of the regular-grid algebra of csrc/geodesic.cu (t = (N + h) cos lat,
    Z = (b^2/a^2 N + h) sin lat, D = lon_k - lon_c; e = t_k sin D, p = t_k cos D - t_c, w = Z_k - Z_c,
    n = cos(lat_c) w - sin(lat_c) p, u = cos(lat_c) p + sin(lat_c) w) -- checked here against the
    oracle, which forms the same quantities through ECEF X, Y, Z like geodesic.py:60-118."""
    a2, b2, inv2r = 6378137.0 ** 2, 6356752.314245 ** 2, 1.0 / (2.0 * 6370994.884953014)
    h_, w_ = z.shape
    la = np.radians(lat)
    s, c = np.sin(la), np.cos(la)
    n_ = a2 / np.sqrt(a2 * c * c + b2 * s * s)
    m_ = b2 / a2 * n_
    dl = np.radians(np.diff(lon))
    sd, cd = np.sin(dl), np.cos(dl)
    out = np.full((h_, w_), np.nan)
    for y in range(1, h_ - 1):
        for x in range(1, w_ - 1):
            h9 = z[y - 1:y + 2, x - 1:x + 2] * zf
            if np.isnan(h9).any():
                continue
            tc, zc = (n_[y] + h9[1, 1]) * c[y], (m_[y] + h9[1, 1]) * s[y]
            es, ns, us = [], [], []
            for dy in range(3):
                for dx in range(3):
                    if dy == 1 and dx == 1:
                        continue
                    r = y + dy - 1
                    t, zz = (n_[r] + h9[dy, dx]) * c[r], (m_[r] + h9[dy, dx]) * s[r]
                    q, e = (t, 0.0) if dx == 1 else ((t * cd[x - 1], -t * sd[x - 1]) if dx == 0 else (t * cd[x], t * sd[x]))
                    p, w = q - tc, zz - zc
                    n = c[y] * w - s[y] * p
                    es.append(e), ns.append(n), us.append(c[y] * p + s[y] * w + (e * e + n * n) * inv2r)
            e, n, u = np.array(es + [0.0]), np.array(ns + [0.0]), np.array(us + [0.0])
            e, n, u = e - e.mean(), n - n.mean(), u - u.mean()
            see, snn, sen, seu, snu = (e * e).sum(), (n * n).sum(), (e * n).sum(), (e * u).sum(), (n * u).sum()
            det = see * snn - sen * sen
            a_, b_ = (0.0, 0.0) if abs(det) < 1e-30 else ((seu * snn - snu * sen) / det, (snu * see - seu * sen) / det)
            m2 = a_ * a_ + b_ * b_
            if not aspect:
                out[y, x] = np.degrees(np.arctan(np.sqrt(m2)))
            elif m2 < 1e-14:
                out[y, x] = -1.0
            else:
                ang = np.degrees(np.arctan2(-a_, -b_))
                out[y, x] = ang + 360.0 if ang < 0 else ang
    return out


@pytest.mark.parametrize("lat0", [-0.5, 40.0, 59.5, 88.0])
def test_geodesic_regular_grid_fold_equals_ecef_form(lat0):
    """The algebraic fold used by the CUDA kernel on regular grids gives the oracle's (= the
    reference's ECEF) numbers on coarse 1-degree grids too, where the longitude step is large."""
    rng = np.random.default_rng(42)
    cases = [np.full((6, 8), 500.0), _tilted("east", 1), _tilted("north", -1), rng.uniform(100, 1000, (10, 10))]
    for z in cases:
        la, lo, lat, lon = _geo_grid(z, lat0, lat0 + 1.0)
        ref = o.geodesic(z, la, lo).astype(np.float64)
        np.testing.assert_allclose(_geodesic_folded(z, lat, lon), ref, rtol=2e-6, atol=1e-7, equal_nan=True)
        refa = o.geodesic(z, la, lo, aspect=True).astype(np.float64)
        gota = _geodesic_folded(z, lat, lon, aspect=True)
        np.testing.assert_array_equal(gota == -1, refa == -1)
        m = ~np.isnan(refa) & (refa != -1)
        d = np.abs(gota[m] - refa[m])
        assert (np.minimum(d, 360 - d) < 1e-4).all()

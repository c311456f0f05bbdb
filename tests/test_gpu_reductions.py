"""The reductions against float64 references at their edges: zonal statistics (zonal_hash_kernel), majority
and the 2-D crosstab (zonal_pair_kernel), the 3-D crosstab, and hotspots (global_stats_kernel,
hotspots_classify_kernel).  Runs on an H100 (`-m gpu`).

The zonal reference is the oracle's numpy two-pass statistics on the values promoted to float64 (cells the
reference skips -- non-finite, or equal to nodata in the values' own dtype -- set to NaN first).  Tolerances:
zone, count, min, max bit-exact; mean within 1e-10 * (|truth| + M), sum within n times that,
1e-10 * (|truth| + n * M); var within 1e-7 * truth + 1e-12 * M^2, std through var; M is the zone's largest
|value| and n its count of valid cells.

Cells whose zone id is not finite belong to no zone.  The reference's sort-and-stride (zonal.py:121-141)
assumes that only NaN ids sort to the end, so a -inf id shifts the values of the zones after it; the truth
here is computed with such ids replaced by NaN."""
import ctypes
import os

import numpy as np
import pytest

import oracle as o
from helpers import K_ZONAL_PAIR, terrain

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

STATS7 = ["mean", "max", "min", "sum", "std", "var", "count"]
H, W = 2002, 2600          # 21 strips of 128 columns (the last one ragged), 8 row segments, H % 4 == 2
FLT_MAX = np.float32(3.4028235e38)
THREADS = os.cpu_count() or 1


@pytest.fixture(scope="module")
def xb():
    import xrspatial_b200
    assert torch.cuda.is_available(), "these tests need a CUDA device"
    return xrspatial_b200


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def da(xb, data):
    return xb.DataArray(data, dims=("y", "x"))


def P(t):
    return ctypes.c_void_p(t.data_ptr())


# ----------------------------------------------------------------- zonal.stats
def truth(zones, values, nodata=None):
    """float64 two-pass statistics of the cells the reference counts, and M per zone."""
    v = np.asarray(values)
    valid = np.isfinite(v)
    if nodata is not None:
        valid &= v != nodata           # numpy compares in the values' dtype (a Python scalar is weak)
    v64 = np.where(valid, v.astype(np.float64), np.nan)
    zones = no_inf_ids(zones)
    ref = o.zonal_stats(zones, v64, stats_funcs=STATS7)
    big = o.zonal_stats(zones, np.abs(v64), stats_funcs=["max"])["max"]
    return ref, big


def no_inf_ids(zones):
    zones = np.asarray(zones)
    return np.where(np.isinf(zones), np.nan, zones).astype(zones.dtype) if zones.dtype.kind == "f" else zones


def check(df, ref, big, what=""):
    got = {c: np.asarray(df[c]) for c in df.columns}
    np.testing.assert_array_equal(got["zone"], ref["zone"], err_msg=what)
    assert got["zone"].dtype == ref["zone"].dtype, what
    for c in ("count", "min", "max"):
        np.testing.assert_array_equal(got[c].astype(np.float64), ref[c], err_msg="%s %s" % (what, c))
    have = ~np.isnan(ref["count"])
    for c in ("mean", "sum", "var", "std"):
        np.testing.assert_array_equal(np.isnan(got[c]), ~have, err_msg="%s %s NaN rows" % (what, c))
    m, n = big[have], ref["count"][have]
    for c, mt in (("mean", m), ("sum", n * m)):
        t, g = ref[c][have], got[c][have]
        err, tol = np.abs(g - t), 1e-10 * (np.abs(t) + mt)
        assert (err <= tol).all(), "%s %s: %d zones out, worst err/tol %.3g" % (what, c, (err > tol).sum(), (err / tol).max())
    tv = ref["var"][have]
    for c, g in (("var", got["var"][have]), ("std", got["std"][have] ** 2)):
        err, tol = np.abs(g - tv), 1e-7 * tv + 1e-12 * m * m
        assert (err <= tol).all(), "%s %s: %d zones out, worst err/tol %.3g (var %g, M %g)" % (
            what, c, (err > tol).sum(), (err / tol).max(), tv[np.argmax(err / tol)], m[np.argmax(err / tol)])


def run(xb, zones, values, nodata=None, what="", stats=STATS7):
    zt, vt = (z if torch.is_tensor(z) else dev(z) for z in (zones, values))
    df = xb.zonal_stats(da(xb, zt), da(xb, vt), stats_funcs=stats, nodata_values=nodata)
    zn = zt.cpu().numpy() if torch.is_tensor(zones) else zones
    vn = vt.cpu().numpy() if torch.is_tensor(values) else values
    ref, big = truth(zn, vn, nodata)
    check(df, ref, big, what)
    return df


def geometries(h, w):
    y, x = np.mgrid[0:h, 0:w]
    band_rows = np.repeat(np.arange(h), np.arange(h) % 5 + 1)[:h]      # bands 1, 2, 3, 4, 5, 1, ... rows high
    stripe_cols = np.repeat(np.arange(w), np.arange(w) % 3 + 1)[:w]    # stripes 1, 2, 3, 1, ... columns wide
    rough = terrain(np.random.default_rng(55), h, w) + np.random.default_rng(56).standard_normal((h, w)) * 60
    return {
        "strip_blocks": (y // 250) * 100 + x // 256,
        "blocks37": (y // 41) * 100 + x // 37,
        "bands": np.broadcast_to(band_rows[:, None], (h, w)),
        "stripes": np.broadcast_to(stripe_cols[None, :], (h, w)),
        "checker": (y + x) % 2,
        "contours": np.floor(rough / 150.0),                              # patchy zones
        "hashed": (y * 7919 + x * 104729) % 4999,
    }


def dirty_values(rng, h, w):
    v = terrain(rng, h, w, nans=0.01)
    n = h * w
    for bad in (np.inf, -np.inf, FLT_MAX, -FLT_MAX):
        v.reshape(-1)[rng.integers(0, n, size=40)] = bad
    return v


GEOMETRIES = ["strip_blocks", "blocks37", "bands", "stripes", "checker", "contours", "hashed"]


@pytest.mark.parametrize("geom", GEOMETRIES)
def test_zonal_geometries(xb, geom):
    rng = np.random.default_rng(100 + GEOMETRIES.index(geom))
    zones = np.ascontiguousarray(geometries(H, W)[geom]).astype(np.int32)
    run(xb, zones, terrain(rng, H, W, nans=0.01), what=geom + " clean")
    run(xb, zones, dirty_values(rng, H, W), what=geom + " +-inf, FLT_MAX")


def test_zonal_against_the_float32_reference(xb):
    """the reference's own float32 statistics, at the tolerance of the rest of the suite"""
    rng = np.random.default_rng(3)
    zones = np.ascontiguousarray(geometries(H, W)["blocks37"]).astype(np.int32)
    values = terrain(rng, H, W, nans=0.01)
    df = xb.zonal_stats(da(xb, dev(zones)), da(xb, dev(values)), stats_funcs=STATS7)
    ref = o.zonal_stats(zones, values, stats_funcs=STATS7)
    np.testing.assert_array_equal(np.asarray(df["zone"]), ref["zone"])
    for c in ("count", "min", "max"):
        np.testing.assert_array_equal(np.asarray(df[c], dtype=np.float64), ref[c], err_msg=c)
    for c in ("mean", "sum", "std", "var"):
        np.testing.assert_allclose(np.asarray(df[c]), ref[c], rtol=1e-5, err_msg=c)


def test_zonal_layouts(xb):
    """ragged widths (W % 4 != 0), bases that are not 16-byte aligned, one row, one column"""
    rng = np.random.default_rng(4)
    for w in (2599, 130):
        g = geometries(H, w)
        for name in ("blocks37", "stripes", "hashed"):
            run(xb, np.ascontiguousarray(g[name]).astype(np.int32), dirty_values(rng, H, w), what="W=%d %s" % (w, name))
    zones = np.ascontiguousarray(geometries(H, W)["blocks37"]).astype(np.int32)
    values = dirty_values(rng, H, W)
    zbuf = torch.empty(H * W + 3, dtype=torch.int32, device="cuda")
    vbuf = torch.empty(H * W + 1, dtype=torch.float32, device="cuda")
    zt = zbuf[3:].view(H, W)
    vt = vbuf[1:].view(H, W)
    zt.copy_(dev(zones))
    vt.copy_(dev(values))
    assert zt.data_ptr() % 16 and vt.data_ptr() % 16 and zt.is_contiguous() and vt.is_contiguous()
    run(xb, zt, vt, what="misaligned bases")
    run(xb, zones[:1], values[:1], what="one row")
    run(xb, np.ascontiguousarray(zones[:, 5:6]), np.ascontiguousarray(values[:, 5:6]), what="one column")
    run(xb, np.ascontiguousarray(zones[:, :3]), np.ascontiguousarray(values[:, :3]), what="three columns")


def _zone_dtype_cases():
    g = geometries(H, W)["blocks37"]
    ids = np.unique(g)
    i32 = np.array([np.iinfo(np.int32).min, np.iinfo(np.int32).max, -1, -7, -123456, 0, 1], np.int64)
    i64 = np.array([np.iinfo(np.int64).min, np.iinfo(np.int64).max, 2 ** 53, 2 ** 53 + 1, 2 ** 53 + 2, 2 ** 60 + 3,
                    -(2 ** 53) - 1, -5, 0], np.int64)
    f = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, -2.5, 1e30, np.nan], np.float64)

    def remap(table, dtype):
        lut = np.concatenate([table, np.arange(len(ids) - len(table), dtype=np.int64) * 3 + 1000]).astype(dtype)
        return np.ascontiguousarray(lut[np.searchsorted(ids, g)])
    return {"int32": remap(i32, np.int32), "int64": remap(i64, np.int64),
            "float32": remap(f, np.float32), "float64": remap(f, np.float64)}


@pytest.mark.parametrize("zdt", ["int32", "int64", "float32", "float64"])
def test_zonal_zone_dtypes(xb, zdt):
    """int32 incl. INT32_MIN / INT32_MAX and negative ids; int64 incl. ids above 2^53 and INT64_MIN (the
    table's empty key); float ids incl. NaN, +-inf (not zones) and -0.0 next to +0.0 (one zone)."""
    rng = np.random.default_rng(11)
    zones = _zone_dtype_cases()[zdt]
    values = np.round(terrain(rng, H, W, nans=0.01) / 16.0).astype(np.float32)    # repeated values: a real majority
    df = run(xb, zones, values, what=zdt, stats=STATS7 + ["majority"])
    if zdt == "int64":
        assert np.iinfo(np.int64).min in set(np.asarray(df["zone"]).tolist())
    maj = o.zonal_stats(no_inf_ids(zones), values, stats_funcs=["majority"])["majority"]
    np.testing.assert_array_equal(np.asarray(df["majority"]), maj, err_msg=zdt + " majority")
    run(xb, zones, values.astype(np.float64) * 1.25 + 1e5, what=zdt + " float64 values")


def test_zonal_nodata_and_invalid_zones(xb):
    """nodata 0.1, which float32 cannot hold: cells equal to float32(0.1) are skipped, like the reference's
    float32 comparison; zones whose cells are all NaN, all inf or all nodata still get a NaN row"""
    rng = np.random.default_rng(12)
    zones = np.ascontiguousarray(geometries(H, W)["blocks37"]).astype(np.int32)
    values = terrain(rng, H, W, nans=0.01)
    values[rng.random(values.shape) < 0.2] = np.float32(0.1)
    values[zones == 5] = np.nan
    values[zones == 6] = np.inf
    values[zones == 7] = np.float32(0.1)
    df = run(xb, zones, values, nodata=0.1, what="nodata 0.1")
    assert np.isnan(np.asarray(df["count"])[np.isin(np.asarray(df["zone"]), [5, 6, 7])]).all()
    run(xb, zones, values.astype(np.float64), nodata=0.1, what="nodata 0.1, float64 values")


@pytest.mark.parametrize("vdt", [np.float32, np.float64])
def test_zonal_zones_far_from_the_pivot(xb, vdt):
    """zones offset by 1e3 .. 1e7 with spreads 0.01 .. 1 next to zones near 0: about one global pivot,
    s2/n - (s1/n)^2 cancels; constant zones have var exactly 0"""
    rng = np.random.default_rng(13)
    zones = np.ascontiguousarray(geometries(H, W)["strip_blocks"]).astype(np.int32)
    ids = np.unique(zones)
    offs = np.array([0.0, 1e3, 1e4, 1e5, 1e6, 3e6, 1e7])
    spreads = np.array([0.01, 0.1, 1.0])
    k = np.searchsorted(ids, zones)
    off = offs[k % len(offs)]
    spread = spreads[(k // len(offs)) % len(spreads)]
    values = (off + spread * rng.standard_normal(zones.shape)).astype(vdt)
    for j, c in enumerate((0.1, 3e6, -7.25, 1e7)):
        values[zones == ids[3 + 5 * j]] = c                      # constant zones
    values[rng.random(values.shape) < 0.01] = np.nan
    df = run(xb, zones, values, what="offsets %s" % np.dtype(vdt).name)
    const = np.isin(np.asarray(df["zone"]), ids[3:20:5])
    assert (np.asarray(df["var"])[const] == 0).all() and (np.asarray(df["std"])[const] == 0).all()


def test_zonal_table_pressure(xb):
    """more distinct zones per CTA than its 1408 slots, more than the 65536 slots of the first global table
    (overflow, retry with a table 16 times larger), and more than 4096 zones with float64 values (the
    second pass gathers the table instead of the packed copy)"""
    rng = np.random.default_rng(14)
    y, x = np.mgrid[0:H, 0:W]
    values = dirty_values(rng, H, W)
    many = ((y * 7919 + x * 104729) % 70001).astype(np.int32)
    df = run(xb, many, values, what="70001 zones")
    assert len(df) == 70001
    spill = ((y * 7919 + x * 104729) % 20011).astype(np.int32)
    run(xb, spill, values, what="20011 scattered zones")
    run(xb, spill, values.astype(np.float64) + 1e4, what="20011 zones, float64 values")


# ----------------------------------------------------------------- majority and crosstab
def _int32_min_raster(rng):
    h, w = 700, 1030
    y, x = np.mgrid[0:h, 0:w]
    zones = ((y // 70) * 10 + x // 103).astype(np.int64)
    zones[(y // 70) % 3 == 0] = np.iinfo(np.int32).min          # the usual int32 nodata id, a large zone
    zones[:, 900:950] = np.iinfo(np.int32).max
    zones[(y < 35) & (x < 103)] = -3
    values = rng.integers(0, 4, size=(h, w)).astype(np.float32)
    values[rng.random(values.shape) < 0.5] *= -1                  # -0.0 next to 0.0
    values[values == 3] = np.nan
    return zones, values


@pytest.mark.parametrize("zdt", [np.int32, np.int64])
def test_majority_and_crosstab_with_the_int32_min_zone(xb, zdt):
    """(INT32_MIN zone, value 0.0) was the pair table's empty key: its counts went to an empty slot"""
    rng = np.random.default_rng(15)
    zones, values = _int32_min_raster(rng)
    zones = zones.astype(zdt)
    for case in ("mixed", "all zeros"):
        v = values.copy()
        if case == "all zeros":
            v[zones == np.iinfo(np.int32).min] = np.where(rng.random(((zones == np.iinfo(np.int32).min).sum(),)) < 0.5,
                                                          np.float32(0.0), np.float32(-0.0))
        df = xb.zonal_stats(da(xb, dev(zones)), da(xb, dev(v)), stats_funcs=["majority", "count"])
        ref = o.zonal_stats(zones, v, stats_funcs=["majority", "count"])
        np.testing.assert_array_equal(np.asarray(df["zone"]), ref["zone"])
        np.testing.assert_array_equal(np.asarray(df["majority"]), ref["majority"], err_msg=case)
        np.testing.assert_array_equal(np.asarray(df["count"]), ref["count"], err_msg=case)
        if case == "all zeros":
            row = np.asarray(df["zone"]) == np.iinfo(np.int32).min
            assert np.asarray(df["majority"])[row][0] == 0.0
        ct = xb.zonal_crosstab(da(xb, dev(zones)), da(xb, dev(v)))
        assert xb._lib.lib().xrs_debug_last_used_tma() == K_ZONAL_PAIR
        rc = o.crosstab(zones, v)
        np.testing.assert_array_equal(np.asarray(ct["zone"]), rc["zone"])
        cats = [c for c in rc if c != "zone"]
        assert [float(c) for c in ct.columns[1:]] == [float(c) for c in cats]
        for c, cc in zip(ct.columns[1:], cats):
            np.testing.assert_array_equal(np.asarray(ct[c]), rc[cc], err_msg="%s crosstab %s" % (case, c))


def test_crosstab_3d_var_std_far_from_the_pivot(xb):
    """3-D crosstab, agg var / std / mean, float32 layers whose zones sit far from the layer's pivot"""
    rng = np.random.default_rng(16)
    h, w = 600, 700
    zones = ((np.arange(h)[:, None] // 100) * 7 + np.arange(w)[None, :] // 100).astype(np.int32)
    offs = np.array([0.0, 1e4, 1e6, 1e7, 3e5])
    layers = []
    for j in range(3):
        off = offs[(zones + j) % len(offs)]
        layers.append((off + 0.1 * (j + 1) * rng.standard_normal((h, w))).astype(np.float32))
    v3 = np.stack(layers)
    v3[rng.random(v3.shape) < 0.01] = np.nan
    vagg = xb.DataArray(dev(v3), dims=("band", "y", "x"))
    vagg["band"] = [10.0, 20.0, 30.0]
    zagg = xb.DataArray(dev(zones), dims=("y", "x"))
    refs = [truth(zones, v3[j]) for j in range(3)]
    for agg in ("var", "std", "mean"):
        df = xb.zonal_crosstab(zagg, vagg, layer=0, agg=agg)
        np.testing.assert_array_equal(np.asarray(df["zone"]), refs[0][0]["zone"])
        for j, c in enumerate((10.0, 20.0, 30.0)):
            ref, big = refs[j]
            g = np.asarray(df[c], dtype=np.float64)
            if agg == "mean":
                tol = 1e-10 * (np.abs(ref["mean"]) + big)
                err = np.abs(g - ref["mean"])
            else:
                g = g ** 2 if agg == "std" else g
                tol = 1e-7 * ref["var"] + 1e-12 * big * big
                err = np.abs(g - ref["var"])
            assert (err <= tol).all(), "%s layer %g: worst err/tol %.3g" % (agg, c, (err / tol).max())


def test_crosstab_3d_columns_are_zonal_stats_of_their_layers(xb, monkeypatch):
    """Every category column of a 3-D crosstab is zonal.stats of that layer with the same zone_ids and nodata,
    its zones in the caller's order with repeats kept.  Layers of float32, float64, float16 and int32 values,
    one of them with zones far from the pivot (the float32 one takes the second pass over a selection), and a zone
    without valid cells (in the int32 raster, with nodata only).  min / max / majority and count exactly, the
    moments within the tolerances of this module: the float64 sums are merged by atomics, so two calls may
    differ in the last bits."""
    from xrspatial_b200 import _lib
    rng = np.random.default_rng(19)
    h, w = 300, 420
    y, x = np.mgrid[0:h, 0:w]
    zones = ((y // 15) * 20 + x // 21).astype(np.int32)                            # 400 zones
    ids = np.unique(zones)
    empty, nodata = ids[7], 5.0
    offs = np.array([0.0, 1e4, 1e6, 1e7, 3e5])                                     # as in the test above
    base = np.stack([np.round(rng.standard_normal((h, w)) * 160) / 4,              # quarter steps: repeated values
                     offs[zones % len(offs)] + 0.1 * rng.standard_normal((h, w)),
                     rng.integers(0, 9, (h, w)).astype(np.float64)])
    sprinkle = rng.random(base.shape) < 0.05
    sprinkle[1] = False                                          # nodata cells would widen the far zones' spread
    base[sprinkle] = nodata
    base[rng.random(base.shape) < 0.01] = np.nan
    base[:, zones == empty] = np.nan
    zagg = xb.DataArray(dev(zones), dims=("y", "x"))
    cats = [1.0, 2.0, 3.0]
    aggs = ("mean", "max", "min", "sum", "std", "var", "count", "majority")
    real_call = _lib.call
    for dt in (np.float32, np.float64, np.float16, np.int32):
        with np.errstate(over="ignore"):                        # float16: the offsets above 65504 become inf
            v3 = (np.where(np.isnan(base), nodata, base) if dt == np.int32 else base).astype(dt)
        vagg = xb.DataArray(dev(v3), dims=("band", "y", "x"))
        vagg["band"] = cats
        for zone_ids in (None, [ids[50], ids[3], empty, ids[50], 10 ** 6, ids[399], ids[0]]):
            want_zones = ids if zone_ids is None else np.array([z for z in zone_ids if z in ids])
            df = xb.zonal_crosstab(zagg, vagg, zone_ids=zone_ids, layer=0, cat_ids=[])
            assert list(df.columns) == ["zone"]
            np.testing.assert_array_equal(np.asarray(df["zone"]), want_zones)
            for nd in (None, nodata):
                what = "%s zone_ids %s nodata %s" % (np.dtype(dt).name, zone_ids is not None, nd)
                layers = [xb.DataArray(dev(v3[j]), dims=("y", "x")) for j in range(len(cats))]
                mm = [xb.zonal_stats(zagg, la, zone_ids=zone_ids, stats_funcs=["min", "max", "count"],
                                     nodata_values=nd) for la in layers]
                for agg in aggs:
                    calls = []
                    monkeypatch.setattr(_lib, "call", lambda name, *a: (calls.append(name), real_call(name, *a))[1])
                    ct = xb.zonal_crosstab(zagg, vagg, zone_ids=zone_ids, layer=0, agg=agg, nodata_values=nd)
                    monkeypatch.setattr(_lib, "call", real_call)
                    if dt == np.float32 and agg == "var" and zone_ids is not None:
                        assert "xrs_zonal_hash_second_pass" in calls, what
                    assert list(ct.columns) == ["zone"] + cats, what
                    zone = np.asarray(ct["zone"])
                    np.testing.assert_array_equal(zone, want_zones, err_msg=what)
                    for j, c in enumerate(cats):
                        st = xb.zonal_stats(zagg, layers[j], zone_ids=zone_ids, stats_funcs=[agg], nodata_values=nd)
                        row = np.searchsorted(np.asarray(st["zone"]), zone)
                        np.testing.assert_array_equal(np.asarray(st["zone"])[row], zone, err_msg=what)
                        t = np.asarray(st[agg], dtype=np.float64)[row]
                        g = np.asarray(ct[c])
                        msg = "%s %s layer %g" % (what, agg, c)
                        if agg == "count":
                            assert g.dtype == np.int64, msg
                            np.testing.assert_array_equal(g, np.where(np.isnan(t), 0, t).astype(np.int64), err_msg=msg)
                            continue
                        if agg in ("min", "max", "majority"):
                            np.testing.assert_array_equal(g, t, err_msg=msg)
                            continue
                        np.testing.assert_array_equal(np.isnan(g), np.isnan(t), err_msg=msg)
                        have = ~np.isnan(t)
                        ref = mm[j]
                        big = np.maximum(np.abs(np.asarray(ref["min"])), np.abs(np.asarray(ref["max"])))[row][have]
                        n = np.asarray(ref["count"], dtype=np.float64)[row][have]
                        g, t = g[have], t[have]
                        if agg == "mean":
                            tol = 1e-10 * (np.abs(t) + big)
                        elif agg == "sum":
                            tol = 1e-10 * (np.abs(t) + n * big)
                        else:
                            if agg == "std":
                                g, t = g ** 2, t ** 2
                            tol = 1e-7 * t + 1e-12 * big * big
                        err = np.abs(g - t)
                        assert (err <= tol).all(), "%s: worst err/tol %.3g" % (msg, (err / tol).max())


# ----------------------------------------------------------------- hotspots
def classify(z):
    t = dev(np.asarray(z, np.float32))
    out = torch.empty(t.numel(), dtype=torch.int8, device=t.device)
    import xrspatial_b200._lib as L
    L.call("xrs_hotspots_classify_f32", P(t), t.numel(), 0.0, 1.0, P(out), ctypes.c_void_p(0))
    return out.cpu().numpy()


def test_hotspots_classification_kernel(xb, refout):
    """gmean 0, gstd 1: z is the input itself.  The reference's classes at the thresholds, then every float32
    in +-[1, 3]"""
    z = refout["hotspots.classify.z"]
    np.testing.assert_array_equal(classify(z), refout["hotspots.classify.out"])
    lo, hi = np.float32(1.0).view(np.int32), np.float32(3.0).view(np.int32)
    pos = np.arange(lo, hi + 1, dtype=np.int32).view(np.float32)
    for zz in (pos, -pos):
        got = classify(zz)
        ref = o.hotspots_classify(zz)
        bad = np.flatnonzero(got != ref)
        assert bad.size == 0, "%d classes differ, first at z = %r" % (bad.size, zz[bad[:3]])


def global_stats(t, pivot):
    import xrspatial_b200._lib as L
    part = torch.empty(3, dtype=torch.float64, device=t.device)
    L.call("xrs_global_stats_f32", P(t), t.numel(), pivot, P(part), ctypes.c_void_p(0))
    return part.cpu().numpy()


def test_global_stats_kernel(xb):
    rng = np.random.default_rng(17)
    for n in (1, 3, 5, (1 << 20) + 3):
        for off, spread in ((0.0, 1000.0), (1e6, 1.0)):
            v = (off + spread * rng.standard_normal(n)).astype(np.float32)
            v[rng.random(n) < 0.01] = np.nan
            buf = torch.empty(n + 1, dtype=torch.float32, device="cuda")
            for t in (dev(v), buf[1:]):                              # aligned (vector loads) and misaligned (scalar)
                t.copy_(dev(v))
                pivot = float(off) + 0.37
                cnt, s1, s2 = global_stats(t, pivot)
                d = v[~np.isnan(v)].astype(np.float64) - pivot
                assert cnt == d.size
                assert abs(s1 - d.sum()) <= 1e-12 * np.abs(d).sum() + 1e-300, (n, off)
                assert abs(s2 - (d * d).sum()) <= 1e-12 * (d * d).sum() + 1e-300, (n, off)


def test_global_stats_kernel_beyond_2_31_cells(xb):
    n = (1 << 31) + 7
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < n * 4 + (1 << 30):
        pytest.skip("needs %.1f GB of free device memory" % (n * 4 / 1e9 + 1))
    t = torch.full((n,), 1.5, dtype=torch.float32, device="cuda")
    t[-1] = 3.5                         # the last cell, beyond 2^31: the 64-bit indexing must reach it
    t[-3] = float("nan")
    t[5] = float("nan")
    cnt, s1, s2 = global_stats(t, 1.0)
    del t
    torch.cuda.empty_cache()
    assert cnt == n - 2
    assert s1 == 0.5 * (n - 3) + 2.5 and s2 == 0.25 * (n - 3) + 6.25


def _disc(r):
    y, x = np.mgrid[-r:r + 1, -r:r + 1]
    return (x * x + y * y <= r * r).astype(np.float64)


@pytest.mark.parametrize("shape", [(4096, 4096), (3001, 2999)])
def test_hotspots_public_vs_oracle(xb, shape):
    """A cell may differ only where the float64 z-score lies within 1e-5 of a threshold (the global mean and std
    are float64 sums here and float32 pairwise sums in the reference)."""
    rng = np.random.default_rng(18)
    h, w = shape
    z = terrain(rng, h, w)
    z[h // 3:h // 3 + 40, w // 4:w // 4 + 50] += 3000.0
    z[2 * h // 3:2 * h // 3 + 30, w // 2:w // 2 + 30] -= 2500.0
    z[rng.random(z.shape) < 0.001] = np.nan
    for kern in (np.ones((5, 5)), _disc(4)):
        got = xb.hotspots(da(xb, dev(z)), kern).data.cpu().numpy()
        ref = o.hotspots(z, kern, nthreads=THREADS)
        mean_array = o.convolve_2d(z, kern / kern.sum(), nthreads=THREADS).astype(np.float64)
        zz = z[~np.isnan(z)].astype(np.float64)
        z64 = np.abs((mean_array - zz.mean()) / zz.std())
        near = np.zeros(z.shape, bool)
        for thr in (1.29, 1.65, 1.96, 2.33, 2.58):
            near |= np.abs(z64 - thr) <= 1e-5
        diff = got != ref
        assert not (diff & ~near).any(), "%d cells differ away from the thresholds" % (diff & ~near).sum()
        assert set(np.unique(ref)) >= {-99, 0, 99}

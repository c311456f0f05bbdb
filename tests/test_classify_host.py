"""classify's host side without a GPU: the public signatures against the reference's, the key image of every
cell type, and the break arithmetic of every scheme reproducing the reference's breaks (golden data from
oracle/make_golden_classify.py) when fed order statistics and moments computed here with NumPy."""
import inspect
import json
import os

import numpy as np
import pytest

import xrspatial_b200 as xb
from xrspatial_b200 import classify as cl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
TOL = 2.0 ** -20      # std_mean / head_tail_breaks: breaks within TOL * max|finite value| (DESIGN.md section 4.11)


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(GOLDEN, "classify_reference.npz"), allow_pickle=False))


def decode(kw):
    return {k: [float(x) if isinstance(x, str) else x for x in v] if isinstance(v, list) else v for k, v in kw.items()}


def golden_calls(g, fns=None):
    for case, fn, kw, tag in json.loads(str(g["calls"])):
        if fns is None or fn in fns:
            yield case, fn, decode(kw), tag


class HostStats:
    """What the schemes read from the device, computed from the finite cells with NumPy."""

    def __init__(self, data):
        self.dtype = data.dtype
        self.v = np.sort(data[np.isfinite(data)])

    def finite_count(self):
        return self.v.size

    def order_stats(self, ranks):
        return self.v[np.asarray(ranks)]

    def moments(self, above=-np.inf):
        x = self.v.astype(np.float64)
        x = x[x > above]
        if x.size == 0:
            return 0, 0.0, 0.0, np.inf, -np.inf
        m = x.mean()
        return x.size, m, float(((x - m) ** 2).sum()), x.min(), x.max()


class HostGaps:
    def __init__(self, data):
        self.dtype = data.dtype
        self.uv = np.unique(data[np.isfinite(data)])

    def unique_count(self):
        return self.uv.size

    def unique_values(self):
        return self.uv

    def largest(self):
        return self.uv[-1]

    def gap_pairs(self, start):
        idx = np.sort(np.argsort(np.diff(self.uv), kind="stable")[start:])
        return self.uv[idx], self.uv[idx + 1]


def host_bins(fn, data, kw):
    st = HostStats(data)
    if fn == "quantile":
        return cl.quantile_bins(st, kw["k"])
    if fn == "percentiles":
        return cl.percentiles_bins(st, kw.get("pct", [1, 10, 50, 90, 99]))
    if fn == "box_plot":
        return cl.box_plot_bins(st, kw.get("hinge", 1.5))
    if fn == "equal_interval":
        return cl.equal_interval_bins(st, kw.get("k", 5))[0]
    if fn == "std_mean":
        return cl.std_mean_bins(st)
    if fn == "head_tail_breaks":
        return cl.head_tail_bins(st)
    if fn == "maximum_breaks":
        return cl.maximum_breaks_bins(HostGaps(data), kw.get("k", 5))
    raise KeyError(fn)


def test_signatures_match_the_reference():
    from make_golden import encode_default
    ref = json.load(open(os.path.join(GOLDEN, "classify_signature.json")))
    assert len(ref) == 9
    for name, params in ref.items():
        fn = getattr(xb, name)
        got = [[k, encode_default(v.default)] for k, v in inspect.signature(inspect.unwrap(fn)).parameters.items()]
        assert got == params, name
        assert getattr(cl, name) is fn


def test_exact_schemes_reproduce_the_reference_breaks(golden):
    n = 0
    for case, fn, kw, tag in golden_calls(golden, {"quantile", "percentiles", "box_plot", "equal_interval",
                                                   "maximum_breaks"}):
        data = golden["case__" + case]
        if "err__" + tag in golden:
            with pytest.raises(Exception) as e:
                host_bins(fn, data, kw)
            assert type(e.value).__name__ == str(golden["err__" + tag]), tag
            continue
        got = host_bins(fn, data, kw)
        want = golden["bins__" + tag]
        assert got.dtype == want.dtype and got.shape == want.shape, tag
        assert np.array_equal(got, want, equal_nan=True), tag
        n += 1
    assert n > 100


def test_mean_schemes_are_within_the_stated_tolerance(golden):
    for case, fn, kw, tag in golden_calls(golden, {"std_mean", "head_tail_breaks"}):
        data = golden["case__" + case]
        if "err__" + tag in golden:
            with pytest.raises(Exception) as e:
                host_bins(fn, data, kw)
            assert type(e.value).__name__ == str(golden["err__" + tag]), tag
            continue
        got, want = host_bins(fn, data, kw), golden["bins__" + tag]
        assert got.shape == want.shape, tag
        fin = data[np.isfinite(data)]
        scale = np.abs(fin).max() if fin.size else 0.0
        assert np.all(np.abs(got - want) <= TOL * scale) or np.array_equal(got, want, equal_nan=True), tag


@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.int16, np.uint16, np.int32, np.int64])
def test_key_image_round_trips_and_orders(dtype):
    """_values inverts the kernels' key: the keys written here the way classify.cu does sort like the values."""
    rng = np.random.default_rng(5)
    if np.dtype(dtype).kind == "f":
        v = np.concatenate([rng.normal(0, 1e3, 500), [0.0, -0.0, 1e-38, -1e-38, 3e38, -3e38]]).astype(dtype)
        bits = np.dtype(dtype).itemsize * 8
        ut = np.dtype("u%d" % (bits // 8))
        u = np.where(v == 0, 0, v).astype(dtype).view(ut)
        top = ut.type(1) << ut.type(bits - 1)
        k = np.where(u & top, ~u, u | top).astype(np.uint64)
    else:
        info = np.iinfo(dtype)
        v = np.concatenate([rng.integers(info.min, info.max, 500, dtype=dtype, endpoint=True),
                            np.array([info.min, info.max, 0, -1 if info.min < 0 else 1], dtype)])
        ut = np.dtype("u%d" % np.dtype(dtype).itemsize)
        k = v.view(ut).astype(np.uint64)
        if info.min < 0:
            k ^= np.uint64(1) << np.uint64(8 * np.dtype(dtype).itemsize - 1)
    back = cl._values(k, np.dtype(dtype))
    assert np.array_equal(back, np.where(v == 0, 0, v).astype(dtype))
    assert np.array_equal(np.argsort(k, kind="stable"), np.argsort(np.where(v == 0, 0, v), kind="stable"))


def test_percentile_restatement_matches_numpy_on_awkward_positions():
    rng = np.random.default_rng(11)
    for dtype in (np.float32, np.float64, np.int16, np.int32):
        for n in (1, 2, 3, 7, 100, 1001):
            a = (rng.normal(0, 1e4, n)).astype(dtype)
            st = HostStats(a)
            for q in ([0, 100], np.arange(1, 100, 3.7), 25, 50.0, 99.9, [33.333, 66.667]):
                got = cl.percentiles_of(st, np.dtype(dtype), [q])[0]
                want = np.percentile(a, q)
                assert np.asarray(got).dtype == np.asarray(want).dtype
                assert np.array_equal(got, want), (dtype, n, q)


def test_unique_gaps_take_np_diff_in_the_cells_own_type():
    """int8 rasters are widened for the kernels; their maximum breaks still come from int8 gaps, which wrap."""
    d = np.array([-128, -120, -100, 60, 70, 127, 5, 60], np.int8).reshape(2, 4)
    for k in (2, 3, 4, 9):
        want = host_bins("maximum_breaks", d, {"k": k})
        got = cl.maximum_breaks_bins(cl._UniqueGaps(np.unique(d)), k)
        assert got.dtype == want.dtype and np.array_equal(got, want), k
    assert not np.array_equal(cl.maximum_breaks_bins(cl._UniqueGaps(np.unique(d)), 3),
                              cl.maximum_breaks_bins(cl._UniqueGaps(np.unique(d.astype(np.int16))), 3))

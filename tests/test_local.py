"""local on the GPU: every golden call of the unmodified reference for numpy and torch Datasets; equality with the
host build of the rule on 4096 x 256 stacks of every cell type (all nine functions), on 4096^2 float32 and uint16
stacks (five functions; the host build is the slow side) and on deep and mixed stacks up to K = 200 at 48 x 40;
combine on 8192^2 against a NumPy restatement; repeated calls, a second stream, untouched inputs and pitched
views; variables on two devices rejected."""
import numpy as np
import pytest

import xrspatial_b200 as xb
from test_local_host import REF_FUNCS, build_host, golden, golden_cases, host_call, run_golden_case, same_key
from test_local_host import same_result

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

STATS = ["sum", "mean", "median", "min", "max", "std"]
OTHERS = ["combine", "lowest_position", "highest_position"] + sorted(REF_FUNCS)
TYPES = ["float16", "float32", "float64", "int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64",
         "bool"]


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    return build_host(str(tmp_path_factory.mktemp("lcg")))


def public_call(fn, raster, func=None, ref_var=None, data_vars=None):
    f = getattr(xb.local, fn)
    if fn == "cell_stats":
        r = f(raster, data_vars, func)
    elif ref_var is not None:
        r = f(raster, ref_var, data_vars)
    else:
        r = f(raster, data_vars)
    out = r.data.cpu().numpy() if torch.is_tensor(r.data) else r.data
    return out, (r.attrs["key"] if fn == "combine" else None)


def on_device(ds_vars):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in ds_vars.items()}


def test_every_golden_call_numpy_and_torch():
    n = 0
    for i, ds_vars, fn, func, ref, dv, want in golden_cases(golden()):
        for vs in (ds_vars, on_device(ds_vars)):
            try:
                run_golden_case(public_call, vs, fn, func, ref, dv, want)
            except AssertionError as e:
                raise AssertionError("golden call %d (%s %s): %s" % (i, fn, func, e)) from None
        n += 1
    assert n > 800


def test_results_are_numpy_for_numpy_and_tensors_for_tensors():
    a = np.arange(12.0).reshape(3, 4)
    for data, kind in (({"a": a, "b": a + 1}, np.ndarray), (on_device({"a": a, "b": a + 1}), torch.Tensor)):
        r = xb.local.combine(xb.Dataset(data))
        assert isinstance(r.data, kind) and r.name is None and set(r.attrs) == {"key"}
        assert isinstance(xb.local.cell_stats(xb.Dataset(data)).data, kind)


def seeded(rng, dt, K, H, W):
    if dt == "bool":
        return [rng.random((H, W)) < 0.5 for _ in range(K)]
    if dt.startswith("float"):
        out = []
        for _ in range(K):
            a = rng.integers(-4, 5, (H, W)).astype(dt)
            m = rng.random((H, W)) < 0.4
            a[m] = (rng.standard_normal(m.sum()) * 100).astype(dt)
            a[(a == 0) & (rng.random((H, W)) < 0.5)] = -0.0
            a[rng.random((H, W)) < 0.01] = np.nan
            out.append(a)
        return out
    info = np.iinfo(dt)
    hi = min(int(info.max), 2 ** 63 - 1)
    pool = np.array([info.min, 0, 1, 2, 3, hi], dtype=dt)
    return [np.where(rng.random((H, W)) < 0.2, pool[rng.integers(0, len(pool), (H, W))],
                     rng.integers(0, 4, (H, W)).astype(dt)) for _ in range(K)]


def check_against_host(host, vs, ref, funcs):
    names = ["v%d" % j for j in range(len(vs))]
    ds = dict(zip(names, vs), ref=ref)
    for fn, func in funcs:
        r = "ref" if fn in REF_FUNCS else None
        dv = names if r is None else None
        want, wkey = host_call(host, fn, xb.Dataset(ds), func, r, dv)
        for data in (ds, on_device(ds)):
            got, key = public_call(fn, xb.Dataset(data), func, r, dv)
            assert same_result(got, want), (fn, func, vs[0].dtype)
            if fn == "combine":
                assert same_key(key, wkey)


ALL = [("cell_stats", f) for f in STATS] + [(f, None) for f in OTHERS]


@pytest.mark.parametrize("dt", TYPES)
def test_large_stacks_of_every_cell_type_equal_the_host_rule(host, dt):
    rng = np.random.default_rng(TYPES.index(dt))
    H, W = 4096, 256
    vs = seeded(rng, dt, 4, H, W)
    ref = rng.integers(-1, 6, (H, W)).astype(np.int16)   # popularity's -2 stays above -D
    check_against_host(host, vs, ref, ALL)


def test_4096_square_stacks_equal_the_host_rule(host):
    rng = np.random.default_rng(7)
    for dt in ("float32", "uint16"):
        vs = seeded(rng, dt, 4, 4096, 4096)
        ref = rng.integers(0, 6, (4096, 4096)).astype(np.uint8)
        check_against_host(host, vs, ref, [("cell_stats", "sum"), ("cell_stats", "max"), ("lowest_position", None),
                                           ("equal_frequency", None), ("rank", None)])


@pytest.mark.parametrize("K", [9, 17, 129, 200])
def test_deep_and_mixed_stacks_equal_the_host_rule(host, K):
    rng = np.random.default_rng(K)
    vs = seeded(rng, "float64", K, 48, 40)
    mixed = [seeded(rng, TYPES[j % len(TYPES)], 1, 48, 40)[0] for j in range(K)]
    ref = rng.integers(-1, K + 3, (48, 40)).astype(np.int32)
    check_against_host(host, vs, ref, ALL)
    check_against_host(host, mixed, ref, ALL)


def _combine_restated(a, b):
    """Ids and keys of combine over two layers of non-negative integer values, restated in NumPy: the distinct
    (a, b) pairs (+-0.0 one value) numbered by first occurrence."""
    fa, fb = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    nan = np.isnan(fa) | np.isnan(fb)
    keyed = fa[~nan] * (fb[~nan].max() + 1) + fb[~nan]   # exact: small integers
    _, first, inverse = np.unique(keyed, return_index=True, return_inverse=True)
    order = np.argsort(first)
    number = np.empty(len(first), np.int64)
    number[order] = np.arange(1, len(first) + 1)
    cells = np.flatnonzero(~nan)
    ids = np.full(fa.shape, np.nan)
    ids[cells] = number[inverse.ravel()]
    reps = cells[first[order]]
    key = {i + 1: t for i, t in enumerate(zip(a.ravel()[reps].tolist(), b.ravel()[reps].tolist()))}
    ids = ids.reshape(a.shape)
    return (ids if nan.any() else ids.astype(np.int64)), key


@pytest.mark.parametrize("distinct", [10, 10 ** 7])
def test_combine_8192_square_equals_a_numpy_restatement(distinct):
    rng = np.random.default_rng(distinct)
    n = 8192
    if distinct == 10:
        a = rng.integers(0, 5, (n, n)).astype(np.float32)
        a[a == 0] = np.where(rng.random((a == 0).sum()) < 0.5, -0.0, 0.0)
        b = rng.integers(0, 2, (n, n)).astype(np.int16)
        a[rng.random((n, n)) < 1e-4] = np.nan
        layers = [a, b]
    else:
        side = int(np.ceil(np.sqrt(distinct)))
        layers = [rng.integers(0, side, (n, n)).astype(np.uint16), rng.integers(0, side, (n, n)).astype(np.float32)]
    want, wkey = _combine_restated(*layers)
    r = xb.local.combine(xb.Dataset(on_device({"a": layers[0], "b": layers[1]})))
    got = r.data.cpu().numpy()
    assert same_result(got, want)
    assert len(r.attrs["key"]) == len(wkey) and (distinct == 10 or len(wkey) > 9 * 10 ** 6)
    assert same_key(r.attrs["key"], wkey) if distinct == 10 else r.attrs["key"] == wkey


def test_repeated_calls_second_stream_untouched_inputs_and_pitched_views():
    rng = np.random.default_rng(3)
    base = [torch.from_numpy(v).cuda() for v in seeded(rng, "float32", 5, 300, 700)]
    ref = torch.from_numpy(rng.integers(0, 7, (300, 700)).astype(np.int32)).cuda()
    ds = dict(("v%d" % j, v) for j, v in enumerate(base))
    ds["ref"] = ref
    before = {k: v.clone() for k, v in ds.items()}
    calls = [("cell_stats", f) for f in STATS] + [(f, None) for f in OTHERS]
    first = {c: public_call(c[0], xb.Dataset(ds), c[1], "ref" if c[0] in REF_FUNCS else None,
                            None if c[0] in REF_FUNCS else list(ds)[:-1]) for c in calls}
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for c, (want, wkey) in first.items():
            got, key = public_call(c[0], xb.Dataset(ds), c[1], "ref" if c[0] in REF_FUNCS else None,
                                   None if c[0] in REF_FUNCS else list(ds)[:-1])
            assert same_result(got, want), c
    s.synchronize()
    for k in ds:
        assert torch.equal(torch.nan_to_num(ds[k], 7.0), torch.nan_to_num(before[k], 7.0)), k
    # pitched views: the same cells inside wider buffers, rows not 16-byte aligned
    wide = {}
    for k, v in ds.items():
        buf = torch.zeros((300, 713), dtype=v.dtype, device=v.device)
        buf[:, 3:703] = v
        wide[k] = buf[:, 3:703]
    for c, (want, wkey) in first.items():
        got, key = public_call(c[0], xb.Dataset(wide), c[1], "ref" if c[0] in REF_FUNCS else None,
                               None if c[0] in REF_FUNCS else list(ds)[:-1])
        assert same_result(got, want), c
        if c[0] == "combine":
            assert key == wkey


def test_variables_on_two_devices_are_refused():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    a = torch.zeros((2, 3), device="cuda:0")
    with pytest.raises(ValueError, match="one device"):
        xb.local.cell_stats(xb.Dataset({"a": a, "b": a.to("cuda:1")}))

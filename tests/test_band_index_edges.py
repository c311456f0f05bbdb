"""The band indices bit for bit against a typed NumPy restatement of the reference's Numba kernels.

ndvi, nbr, nbr2, ndmi, savi, evi, arvi, gci, sipi and ebbi (csrc/multispectral.cu) claim bit-identical results
to the reference's `_*_cpu` kernels.  The restatement below computes every sub-expression in the type Numba gives
it (float32 steps in float32, promoted steps in float64, the store rounded to float32); NumPy's float32 add, sub,
mul, div and sqrt are correctly rounded, so it is exact.  The CPU tests pin it against goldens made from the
reference's own kernels (tests/golden/multispectral_edges.npz, oracle/make_golden_multispectral.py) and show
that the goldens see every wrongly typed step.  The GPU tests hold the public functions to it: special values,
zero denominators, the scalar types savi and evi accept, every float4 tail length, misaligned, transposed and
broadcast views, every cell type on numpy and torch containers, rasters on which each thread loops more than
once, and a raster beyond 2^31 cells.

Cells are compared as uint32 bits, so the sign of zero counts; NaN masks must match, NaN payloads need not.
"""
import os

import numpy as np
import pytest

from test_oracle_golden import MS_QGIS

torch = pytest.importorskip("torch")

F, D = np.float32, np.float64
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "multispectral_edges.npz")

# public function -> reference kernel
KERNEL = {"ndvi": "normalized_ratio", "nbr": "normalized_ratio", "nbr2": "normalized_ratio",
          "ndmi": "normalized_ratio", "savi": "savi", "evi": "evi", "arvi": "arvi", "gci": "gci", "sipi": "sipi",
          "ebbi": "ebbi"}
NBANDS = {"normalized_ratio": 2, "savi": 2, "evi": 3, "arvi": 3, "gci": 2, "sipi": 3, "ebbi": 3}
PUBLIC = sorted(KERNEL)
DEFAULTS = {"savi": (1.0,), "evi": (6.0, 7.5, 1.0, 2.5)}

# Soil-factor types for which Numba sums savi's `nir + red + soil_factor` in float32 (measured on the reference,
# pinned by the `savi_type` goldens); every other accepted type sums in float64.
SAVI_F32_SUM = (np.float32, np.int8, np.int16, np.uint8, np.bool_, bool)


# ------------------------------------------------------------------------------------------------ restatement
class Typed(object):
    """Runs named steps in their reference types.  A step computes in the wider of its own type and its operand
    types, and stores in its own type; `mut` flips one step's type (float32 <-> float64)."""

    def __init__(self, mut, **types):
        assert mut is None or mut in types, mut
        self.mut, self.types = mut, types

    def __call__(self, name, fn, *xs):
        t = self.types[name]
        if name == self.mut:
            t = D if t is F else F
        xs = [np.asarray(x) for x in xs]
        ct = np.result_type(t, *[x.dtype for x in xs])
        return fn(*[x.astype(ct) for x in xs]).astype(t)


def _store(q, den):
    """out = q where den != 0 else NaN, as float32 (the reference's `np.full(nan)` and store)."""
    return np.where(den != 0, q, np.nan).astype(F)


def normalized_ratio(a, b, mut=None):
    s = Typed(mut, num=F, den=F, q=F)
    num = s("num", np.subtract, a, b)
    den = s("den", np.add, a, b)
    return _store(s("q", np.divide, num, den), den)


def savi(nir, red, L, mut=None):
    L = np.asarray(L)
    s = Typed(mut, num=F, nr=F, soma=F if isinstance(L[()], SAVI_F32_SUM) else D, onep=D, den=D, q=D)
    num = s("num", np.subtract, nir, red)
    soma = s("soma", np.add, s("nr", np.add, nir, red), L)
    den = s("den", np.multiply, soma, s("onep", np.add, D(1.0), L))
    return _store(s("q", np.divide, num, den), den)


def evi(nir, red, blue, c1, c2, L, G, mut=None):
    s = Typed(mut, num=F, t1=D, t2=D, t3=D, t4=D, den=D, q=D, g=D)
    num = s("num", np.subtract, nir, red)
    t2 = s("t2", np.add, nir, s("t1", np.multiply, np.asarray(c1), red))
    t4 = s("t4", np.subtract, t2, s("t3", np.multiply, np.asarray(c2), blue))
    den = s("den", np.add, t4, np.asarray(L))
    q = s("q", np.divide, num, den)
    return _store(s("g", np.multiply, np.asarray(G), q), den)


def arvi(nir, red, blue, mut=None):
    s = Typed(mut, r2=D, s1=D, num=D, d1=D, den=D, q=D)
    r2 = s("r2", np.multiply, D(2.0), red)
    num = s("num", np.add, s("s1", np.subtract, nir, r2), blue)
    den = s("den", np.add, s("d1", np.add, nir, r2), blue)
    return _store(s("q", np.divide, num, den), den)


def gci(nir, green, mut=None):
    s = Typed(mut, q=F, r=D)
    q = s("q", np.divide, nir, green)
    return _store(s("r", np.subtract, q, D(1.0)), green)


def sipi(nir, red, blue, mut=None):
    s = Typed(mut, num=F, den=F, q=F)
    num = s("num", np.subtract, nir, blue)
    den = s("den", np.subtract, nir, red)
    return _store(s("q", np.divide, num, den), den)


def ebbi(red, swir, tir, mut=None):
    s = Typed(mut, num=F, st=F, sq=F, den=D, q=D)
    num = s("num", np.subtract, swir, red)
    den = s("den", np.multiply, D(10.0), s("sq", np.sqrt, s("st", np.add, swir, tir)))
    return _store(s("q", np.divide, num, den), den)


RESTATED = {"normalized_ratio": normalized_ratio, "savi": savi, "evi": evi, "arvi": arvi, "gci": gci,
            "sipi": sipi, "ebbi": ebbi}
# every step whose result feeds another operation (the last one's type cannot change the stored float32: one
# correctly rounded operation rounded again to float32 is the float32 operation)
STEPS = {"normalized_ratio": ["num", "den"], "savi": ["num", "nr", "soma", "onep", "den"],
         "evi": ["num", "t1", "t2", "t3", "t4", "den", "q"], "arvi": ["r2", "s1", "num", "d1", "den"],
         "gci": ["q"], "sipi": ["num", "den"], "ebbi": ["num", "st", "sq", "den"]}


def restate(kernel, bands, scalars=(), mut=None):
    with np.errstate(all="ignore"):
        bands = [np.asarray(b).astype(F) for b in bands]
        return RESTATED[kernel](*bands, *scalars, mut=mut)


def bit_mismatches(got, want):
    """Cells where got and want differ: NaN in one only, or different float32 bits where neither is NaN."""
    got, want = np.asarray(got, F), np.asarray(want, F)
    assert got.shape == want.shape, (got.shape, want.shape)
    gn, wn = np.isnan(got), np.isnan(want)
    return (gn != wn) | (~gn & ~wn & (got.view(np.uint32) != want.view(np.uint32)))


def assert_bits(got, want, what):
    bad = bit_mismatches(got, want)
    if bad.any():
        i = np.flatnonzero(bad.ravel())[0]
        raise AssertionError("%s: %d of %d cells differ; first at %d: got %r, want %r" % (
            what, int(bad.sum()), bad.size, i, np.asarray(got).ravel()[i], np.asarray(want).ravel()[i]))


# ---------------------------------------------------------------------------------------------------- goldens
def scalar(kind, v):
    if kind in ("float", "int", "bool"):
        return {"float": float, "int": int, "bool": bool}[kind](v)
    return getattr(np, kind)(v)


def golden_cases():
    """(kernel, label, scalars, bands, out) for every case of the goldens."""
    g = np.load(GOLDEN, allow_pickle=False)
    off = g["off"]
    cases = []
    for i, k in enumerate(g["kernel"]):
        kinds = [t for t in str(g["scalar_kinds"][i]).split(",") if t]
        sc = tuple(scalar(t, v) for t, v in zip(kinds, g["scalar_values"][i]))
        lo, hi = off[i], off[i + 1]
        cases.append((str(k), str(g["label"][i]), sc, g["bands"][:NBANDS[str(k)], lo:hi], g["out"][lo:hi]))
    return cases


CASES = golden_cases()


def _case_id(c):
    return "%s-%s-%s" % (c[0], c[1], ",".join("%s(%r)" % (type(s).__name__, s) for s in c[2]))


def test_goldens_cover_what_they_claim():
    kinds = {(c[0], c[1]) for c in CASES}
    for k in NBANDS:
        assert (k, "special") in kinds and (k, "random") in kinds, k
    savi_types = {type(c[2][0]) for c in CASES if c[1] == "savi_type"}
    assert {float, int, bool, np.float32, np.float64, np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16,
            np.uint32, np.uint64, np.bool_} <= savi_types
    # where L is neither 0 nor -1 (which zeroes 1 + L), the float32 sums of the table differ from a float64 sum
    f32 = [c for c in CASES if c[1] == "savi_type" and isinstance(c[2][0], SAVI_F32_SUM) and c[2][0] not in (0, -1)]
    assert f32 and all(bit_mismatches(c[4], restate("savi", c[3], (float(c[2][0]),))).any() for c in f32)


@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_restatement_matches_the_reference(case):
    k, _, sc, bands, out = case
    assert_bits(restate(k, bands, sc), out, _case_id(case))


@pytest.mark.parametrize("kernel,step", [(k, s) for k in STEPS for s in STEPS[k]])
def test_goldens_see_every_wrongly_typed_step(kernel, step):
    """Keeping one float32 step in float64 into the next operation, or rounding one float64 step to float32,
    changes some golden cell."""
    seen = 0
    for k, _, sc, bands, out in CASES:
        if k == kernel:
            seen += int(bit_mismatches(restate(k, bands, sc, mut=step), out).sum())
    assert seen > 0, "%s with %s retyped matches every golden" % (kernel, step)


# -------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def xb():
    import xrspatial_b200
    assert torch.cuda.is_available(), "these tests need a CUDA device"
    return xrspatial_b200


def run(xb, fn, bands, scalars=()):
    """The public function on bands already in their container; the result as a host float32 array."""
    aggs = [xb.DataArray(b, dims=("y", "x")) for b in bands]
    out = getattr(xb, fn)(*aggs, *scalars).data
    if hasattr(out, "cpu"):
        assert out.dtype == torch.float32
        return out.cpu().numpy()
    assert isinstance(out, np.ndarray) and out.dtype == np.float32
    return out


def on(container, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda() if container == "torch" else np.ascontiguousarray(a)


def check(xb, fn, bands, scalars=(), what="", host_bands=None):
    """fn on `bands` against the restatement of the same cells cast to float32."""
    hb = host_bands if host_bands is not None else [
        b.cpu().numpy() if hasattr(b, "cpu") else np.asarray(b) for b in bands]
    got = run(xb, fn, bands, scalars)
    assert_bits(got, restate(KERNEL[fn], hb, scalars), "%s %s" % (fn, what))


def pool(rng, n):
    """n cells drawn from the goldens' bands (special values, zero denominators, rounding-sensitive values)."""
    g = np.load(GOLDEN, allow_pickle=False)["bands"]
    return g[:, rng.integers(0, g.shape[1], n)]


@pytest.mark.gpu
@pytest.mark.parametrize("container", ["torch", "numpy"])
def test_golden_cases_on_device(xb, container):
    for k, label, sc, bands, out in CASES:
        fns = [f for f in PUBLIC if KERNEL[f] == k]
        for fn in fns:
            got = run(xb, fn, [on(container, b.reshape(1, -1)) for b in bands], sc)
            assert_bits(got.ravel(), out, "%s %s %s %r" % (container, fn, label, sc))


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(MS_QGIS))
def test_known_answers_on_device(xb, known, name):
    # the reference's test_multispectral.py QGIS tables, at its tolerance (see test_oracle_golden.py)
    _, bands = MS_QGIS[name]
    for container in ("torch", "numpy"):
        got = run(xb, name, [on(container, known["multispectral.%s_data" % b]) for b in bands])
        np.testing.assert_allclose(got, known["multispectral.qgis_" + name], rtol=1e-5, atol=1e-7, equal_nan=True,
                                   err_msg="%s %s" % (container, name))


@pytest.mark.gpu
def test_uint16_known_answers_on_device(xb, known):
    g = lambda n, i: known["multispectral.uint_%s.%d" % (n, i)]  # noqa: E731
    for fn, kernel, nb in (("ndvi", "normalized_ratio", 2), ("arvi", "arvi", 3), ("evi", "evi", 3),
                           ("savi", "savi", 2), ("sipi", "sipi", 3), ("ebbi", "ebbi", 3)):
        assert g(kernel, 0).dtype == np.uint16
        for container in ("torch", "numpy"):
            got = run(xb, fn, [on(container, g(kernel, i)) for i in range(nb)])
            np.testing.assert_allclose(got, g(kernel, nb), rtol=1e-6, err_msg="%s %s" % (container, fn))


SHAPES = [(1, 1), (1, 2), (1, 3), (1, 4), (1, 5), (1, 7), (1, 8), (1, 9), (3, 5), (5, 6), (7, 7), (6, 11),
          (9, 11), (13, 17)]


@pytest.mark.gpu
@pytest.mark.parametrize("fn", PUBLIC)
def test_every_float4_tail_length(xb, fn):
    rng = np.random.default_rng(1)
    nb = NBANDS[KERNEL[fn]]
    for shape in SHAPES:
        bands = [b.reshape(shape) for b in pool(rng, shape[0] * shape[1])[:nb]]
        for container in ("torch", "numpy"):
            check(xb, fn, [on(container, b) for b in bands], DEFAULTS.get(fn, ()), "%s %s" % (shape, container))


@pytest.mark.gpu
@pytest.mark.parametrize("fn", PUBLIC)
def test_misaligned_row_offset_views(xb, fn):
    """One band is rows 1.. of a buffer whose rows are not a multiple of 16 bytes, so its pointer is not 16-byte
    aligned and the kernel takes its scalar loop; every band in turn."""
    rng = np.random.default_rng(2)
    nb = NBANDS[KERNEL[fn]]
    for H, W in ((1, 5), (4, 7), (33, 37), (64, 1030)):
        bands = [b.reshape(H, W) for b in pool(rng, H * W)[:nb]]
        for j in range(nb):
            big = torch.from_numpy(np.vstack([np.full((1, W), 7.0e3, F), bands[j]])).cuda()
            view = big[1:]
            assert view.is_contiguous() and view.data_ptr() % 16 != 0
            dev = [view if i == j else on("torch", b) for i, b in enumerate(bands)]
            check(xb, fn, dev, DEFAULTS.get(fn, ()), "%dx%d band %d offset" % (H, W, j), host_bands=bands)


@pytest.mark.gpu
@pytest.mark.parametrize("fn", PUBLIC)
def test_transposed_and_broadcast_views(xb, fn):
    rng = np.random.default_rng(3)
    nb = NBANDS[KERNEL[fn]]
    H, W = 21, 13
    bands = [b.reshape(W, H) for b in pool(rng, H * W)[:nb]]
    dev = [on("torch", b).t() for b in bands]
    assert not dev[0].is_contiguous()
    check(xb, fn, dev, DEFAULTS.get(fn, ()), "transposed", host_bands=[b.T for b in bands])
    check(xb, fn, [b.T for b in bands], DEFAULTS.get(fn, ()), "transposed numpy", host_bands=[b.T for b in bands])
    rows = pool(rng, W)[:nb]
    dev = [on("torch", r.reshape(1, W)).expand(H, W) for r in rows]
    assert dev[0].stride(0) == 0
    host = [np.broadcast_to(r.reshape(1, W), (H, W)) for r in rows]
    check(xb, fn, dev, DEFAULTS.get(fn, ()), "broadcast", host_bands=host)
    check(xb, fn, host, DEFAULTS.get(fn, ()), "broadcast numpy", host_bands=host)
    mixed = [dev[0]] + [on("torch", np.ascontiguousarray(h)) for h in host[1:]]
    check(xb, fn, mixed, DEFAULTS.get(fn, ()), "one broadcast band", host_bands=host)


@pytest.mark.gpu
@pytest.mark.parametrize("fn", PUBLIC)
def test_every_thread_loops_more_than_once(xb, fn):
    """More than sm_count * 8 CTAs * 256 threads * 4 cells plus a tail: the float4 loop and the scalar loop (one
    band a cell past alignment) both wrap."""
    import ctypes
    n_sm = ctypes.c_int(0)
    xb._lib.call("xrs_device_sm_count", 0, ctypes.byref(n_sm))
    threads = n_sm.value * 8 * 256
    W = 1031
    H = (2 * threads * 4) // W + 1
    rng = np.random.default_rng(4)
    nb = NBANDS[KERNEL[fn]]
    bands = [b.reshape(H, W) for b in pool(rng, H * W)[:nb]]
    assert H * W > 2 * threads * 4 and (H * W) % 4
    want = restate(KERNEL[fn], bands, DEFAULTS.get(fn, ()))
    dev = [on("torch", b) for b in bands]
    assert_bits(run(xb, fn, dev, DEFAULTS.get(fn, ())), want, fn + " float4")
    flat = torch.empty(H * W + 1, dtype=torch.float32, device="cuda")
    flat[1:] = dev[0].reshape(-1)
    dev[0] = flat[1:].view(H, W)
    assert dev[0].data_ptr() % 16 != 0
    assert_bits(run(xb, fn, dev, DEFAULTS.get(fn, ())), want, fn + " scalar")


def typed_band(rng, dtype, n):
    """n cells of `dtype` across its range: values float32 rounds, extremes, and for floats inf, NaN, -0 and
    values beyond float32's range."""
    dt = np.dtype(dtype)
    if dt == np.bool_:
        return rng.random(n) < 0.5
    if dt.kind in "iu":
        info = np.iinfo(dt)
        v = rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)
        v[:4] = [info.min, info.max, 0, info.max - 1]
        return v
    lo, hi = (-46.0, 39.0) if dt == np.float64 else (-7.0, 4.8)
    v = rng.choice([-1.0, 1.0], n) * 10.0 ** rng.uniform(lo, hi, n)
    v[:6] = [np.inf, -np.inf, np.nan, -0.0, 0.0, 1.0]
    if dt == np.float64:
        v[6:9] = [1e300, -1e-300, float(np.finfo(F).max) * (1 + 2.0 ** -25)]
    return v.astype(dt)


CELL_TYPES = [np.float64, np.float16, np.int16, np.uint16, np.int32, np.int64, np.uint8, np.bool_]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", CELL_TYPES, ids=lambda d: np.dtype(d).name)
@pytest.mark.parametrize("fn", ["ndvi", "savi", "evi", "arvi", "gci", "sipi", "ebbi"])
def test_cell_types(xb, fn, dtype):
    """Bands of every cell type, cast to float32 as `astype('f4')` casts them, on numpy and torch."""
    rng = np.random.default_rng(5)
    nb = NBANDS[KERNEL[fn]]
    bands = [typed_band(rng, dtype, 999).reshape(27, 37) for _ in range(nb)]
    for container in ("torch", "numpy"):
        check(xb, fn, [on(container, b) for b in bands], DEFAULTS.get(fn, ()), container, host_bands=bands)


@pytest.mark.gpu
@pytest.mark.parametrize("fn", ["ndvi", "savi", "evi", "ebbi"])
def test_bfloat16_and_mixed_cell_types(xb, fn):
    rng = np.random.default_rng(6)
    nb = NBANDS[KERNEL[fn]]
    src = pool(rng, 31 * 29)[:nb]
    dev = [torch.from_numpy(b.reshape(31, 29)).cuda().to(torch.bfloat16) for b in src]
    check(xb, fn, dev, DEFAULTS.get(fn, ()), "bfloat16", host_bands=[d.float().cpu().numpy() for d in dev])
    mixed = [typed_band(rng, t, 31 * 29).reshape(31, 29) for t in (np.uint16, np.float64, np.int8)[:nb]]
    for container in ("torch", "numpy"):
        check(xb, fn, [on(container, b) for b in mixed], DEFAULTS.get(fn, ()), "mixed " + container,
              host_bands=mixed)
    dev = [on("torch", mixed[0]).to(torch.bfloat16)] + [on("torch", b) for b in mixed[1:]]
    check(xb, fn, dev, DEFAULTS.get(fn, ()), "bfloat16 with others",
          host_bands=[dev[0].float().cpu().numpy()] + mixed[1:])


@pytest.mark.gpu
def test_ndvi_beyond_2_31_cells(xb):
    """ndvi on two bands of 32769 x 65537 cells (2^31 + 98305, n % 4 == 1), filled on the device in chunks from
    a = ((i mod 1021) + 1) / 4, b = ((i mod 1019) - 509) / 8, once aligned and once as a view one cell into the
    same allocations (the scalar loop).  Compared on the first 2^20 cells and on every cell from 2^31 - 2^20 to
    the end; about 26 GB of device memory."""
    H, W = 32769, 65537
    n = H * W
    need = 3 * 4 * (n + 1) + (1 << 30)
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip("needs %.1f GB of free device memory, %.1f GB free" % (need / 1e9, free / 1e9))
    a = torch.empty(n + 1, dtype=torch.float32, device="cuda")
    b = torch.empty(n + 1, dtype=torch.float32, device="cuda")
    step = 1 << 26
    for s in range(0, n + 1, step):
        i = torch.arange(s, min(s + step, n + 1), dtype=torch.int64, device="cuda")
        a[s:s + i.numel()] = ((i % 1021) + 1).to(torch.float32) * 0.25
        b[s:s + i.numel()] = ((i % 1019) - 509).to(torch.float32) * 0.125
        del i
    # the last window holds the cells around 2^31, the last 2^20 cells, the last float4 group and the tail
    windows = [(0, 1 << 20), (2 ** 31 - (1 << 20), n)]

    def want(lo, hi, shift):
        i = np.arange(lo + shift, hi + shift, dtype=np.int64)
        return restate("normalized_ratio", [((i % 1021) + 1).astype(F) * F(0.25),
                                            ((i % 1019) - 509).astype(F) * F(0.125)])

    try:
        for shift in (0, 1):
            va, vb = a[shift:shift + n].view(H, W), b[shift:shift + n].view(H, W)
            assert (va.data_ptr() % 16 == 0) == (shift == 0)
            out = xb.ndvi(xb.DataArray(va, dims=("y", "x")), xb.DataArray(vb, dims=("y", "x"))).data
            assert out.shape == (H, W) and out.dtype == torch.float32
            flat = out.reshape(-1)
            for lo, hi in windows:
                got = flat[lo:hi].cpu().numpy()
                assert np.isnan(got).any()
                assert_bits(got, want(lo, hi, shift), "shift %d cells [%d, %d)" % (shift, lo, hi))
            del out, flat
    finally:
        del a, b
        torch.cuda.empty_cache()

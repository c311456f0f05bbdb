"""perlin and generate_terrain: noise_octave.cuh compiled for the host -- NumPy's permutation, the warp chunk rule
of the draws and the reservation rounds of the shuffle against the sequential shuffle, and a host restatement of
the noise against the unmodified reference's outputs -- the argument rules and the C entry points' checks; on the
GPU the device tables against NumPy, the reference's outputs, bit equality with the host restatement up to 8192^2,
containers, streams, views and repeated calls."""
import ctypes
import importlib
import inspect
import json
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "xarray-spatial_b200", "csrc", "noise_octave.cuh")
GOLDEN = os.path.join(ROOT, "tests", "golden")
N = 2 ** 20
SEED_LIST = [0, 1, 5] + list(range(10, 26)) + [2 ** 31, 2 ** 32 - 1]
F32_TOL, F64_TOL = 8 * 2.0 ** -24, 16 * 2.0 ** -53   # of the final terrain, times zfactor


def _mod(name):
    return importlib.import_module("xrspatial_b200." + name)


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(GOLDEN, "terrain_reference.npz"), allow_pickle=False))


# ----------------------------------------------------------------------------- the header on the host
@pytest.fixture(scope="module")
def host(tmp_path_factory):
    d = tmp_path_factory.mktemp("nz")
    cpp, so = str(d / "n.cpp"), str(d / "n.so")
    with open(cpp, "w") as f:
        f.write('#include "%s"\n' % HEADER + r"""
#include <algorithm>
#include <vector>
using namespace xrs::nz;
// RandomState(seed).permutation(n).  chunked: the draws by the warp chunk rule (a warp's 32 lanes simulated);
// reserved: the swaps by rounds of reservations.  Returns the number of rounds (0 for sequential swaps) and the
// words drawn in *words; J (n int32) receives each step's draw.
extern "C" long long nz_perm(uint32_t seed, int64_t n, int chunked, int reserved, int32_t *A, int32_t *J,
                             long long *words) {
    uint32_t mt[kMtN];
    mt_init(mt, seed);
    int pos = kMtN;
    auto next = [&]() { if (pos == kMtN) { mt_twist(mt); pos = 0; } return mt_temper(mt[pos++]); };
    uint32_t i = (uint32_t)(n - 1);
    long long used = 0;
    while (i > 0) {
        if (!chunked) { draw(i, next(), J); ++used; continue; }
        uint32_t v[32];
        for (int l = 0; l < 32; ++l) v[l] = next();
        bool fast = chunk_uniform(i);
        for (int l = 0; l < 32 && fast; ++l) fast = !undecided(v[l] & interval_mask(i), i);
        if (fast) {
            int acc = 0;
            const uint32_t m = interval_mask(i);
            for (int l = 0; l < 32; ++l)
                if (sure_accept(v[l] & m, i)) { J[i - acc] = (int32_t)(v[l] & m); ++acc; }
            i -= acc;
            used += 32;
        } else {
            for (int l = 0; l < 32 && i > 0; ++l) { draw(i, v[l], J); ++used; }
        }
    }
    *words = used;
    for (int64_t k = 0; k < n; ++k) A[k] = (int32_t)k;
    if (!reserved) {
        for (int64_t k = n - 1; k >= 1; --k) std::swap(A[k], A[J[k]]);
        return 0;
    }
    std::vector<uint64_t> R(n, 0);
    std::vector<int64_t> pend, next_pend;
    for (int64_t k = n - 1; k >= 1; --k) pend.push_back(k);
    long long rounds = 0;
    while (!pend.empty()) {
        const uint32_t r = (uint32_t)++rounds;
        std::reverse(pend.begin(), pend.end());   // the order of the writes must not matter
        for (int64_t k : pend) {
            const uint64_t key = reservation(r, (uint32_t)k);
            R[k] = std::max(R[k], key);
            R[J[k]] = std::max(R[J[k]], key);
        }
        next_pend.clear();
        for (int64_t k : pend) {
            const uint64_t key = reservation(r, (uint32_t)k);
            if (R[k] == key && R[J[k]] == key) std::swap(A[k], A[J[k]]);
            else next_pend.push_back(k);
        }
        pend.swap(next_pend);
    }
    return rounds;
}
// The field before normalisation, as the kernels compute it: perlin (terrain 0) or the terrain after the cube;
// pre receives the terrain's field before the cube.  stats: 5 int32 per octave, as xrs_noise writes them.
template <typename T>
static void field(const int32_t *tables, const float *xs, int64_t W, const float *ys, int64_t H, int64_t r0,
                  int64_t nr, int terrain, const T *in, T *pre, T *out, int32_t *stats) {
    const int n_oct = terrain ? kTerrainOctaves : 1;
    std::vector<Col> cols(n_oct * W);
    std::vector<Row> rows(n_oct * H);
    for (int o = 0; o < n_oct; ++o) {
        int32_t *st = stats + 5 * o;
        st[0] = 0; st[1] = INT32_MAX; st[2] = INT32_MIN; st[3] = INT32_MAX; st[4] = INT32_MIN;
        for (int64_t j = 0; j < W; ++j) {
            bool ok;
            const Col c = make_col(tables + o * kTableN, octave_coord(xs[j], o), ok);
            cols[o * W + j] = c;
            if (!ok) st[0] = 1;
            else { st[1] = std::min({st[1], c.p0, c.p1}); st[2] = std::max({st[2], c.p0, c.p1}); }
        }
        for (int64_t i = 0; i < H; ++i) {
            bool ok;
            const Row r = make_row(octave_coord(ys[i], o), ok);
            rows[o * H + i] = r;
            if (!ok) st[0] = 1;
            else { st[3] = std::min(st[3], r.yi); st[4] = std::max(st[4], r.yi); }
        }
    }
    for (int64_t i = r0; i < r0 + nr; ++i)
        for (int64_t j = 0; j < W; ++j) {
            const int64_t k = (i - r0) * W + j;
            T h = terrain ? in[k] * (T)0 : (T)0;
            for (int o = 0; o < n_oct; ++o) {
                const double a = octave(tables + o * kTableN, cols[o * W + j], rows[o * H + i]);
                h = terrain ? terrain_add(h, a, octave_weight(o)) : (T)a;
            }
            if (terrain) { pre[k] = terrain_scale(h); out[k] = terrain_cube(pre[k]); }
            else out[k] = h;
        }
}
extern "C" void nz_field_f32(const int32_t *t, const float *xs, int64_t W, const float *ys, int64_t H, int64_t r0,
                             int64_t nr, int terrain, const float *in, float *pre, float *out, int32_t *st) {
    field<float>(t, xs, W, ys, H, r0, nr, terrain, in, pre, out, st);
}
extern "C" void nz_field_f64(const int32_t *t, const float *xs, int64_t W, const float *ys, int64_t H, int64_t r0,
                             int64_t nr, int terrain, const double *in, double *pre, double *out, int32_t *st) {
    field<double>(t, xs, W, ys, H, r0, nr, terrain, in, pre, out, st);
}
""")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, cpp])
    lib = ctypes.CDLL(so)
    I, I64, P = ctypes.c_int, ctypes.c_int64, ctypes.c_void_p
    lib.nz_perm.argtypes = [ctypes.c_uint32, I64, I, I, P, P, ctypes.POINTER(ctypes.c_longlong)]
    lib.nz_perm.restype = ctypes.c_longlong
    for fn in (lib.nz_field_f32, lib.nz_field_f64):
        fn.argtypes = [P, P, I64, P, I64, I64, I64, I, P, P, P, P]
    return lib


def host_perm(lib, seed, n, chunked=False, reserved=False):
    a, j = np.empty(n, np.int32), np.zeros(max(n, 1), np.int32)
    words = ctypes.c_longlong()
    rounds = lib.nz_perm(seed, n, int(chunked), int(reserved), a.ctypes.data, j.ctypes.data, ctypes.byref(words))
    return a, j, words.value, rounds


_TABLES = {}


def tables_of(seeds):
    for s in seeds:
        if s not in _TABLES:
            _TABLES[s] = np.random.RandomState(s).permutation(N).astype(np.int32)
    return np.ascontiguousarray(np.stack([_TABLES[s] for s in seeds]))


def host_field(lib, seeds, xs, ys, terrain, data=None, rows=None):
    """(pre-cube field or None, field before normalisation, stats) of rows [r0, r0 + nr) (default all)."""
    t = tables_of(seeds)
    xs = np.ascontiguousarray(xs, np.float32)
    ys = np.ascontiguousarray(ys, np.float32)
    H, W = len(ys), len(xs)
    r0, nr = rows if rows is not None else (0, H)
    dt = np.float32 if data is None or data.dtype == np.float32 else np.float64
    inp = np.ascontiguousarray(data[r0:r0 + nr] if data is not None else np.zeros((nr, W)), dt)
    pre, out = np.empty((nr, W), dt), np.empty((nr, W), dt)
    st = np.empty((len(seeds), 5), np.int32)
    fn = lib.nz_field_f32 if dt == np.float32 else lib.nz_field_f64
    fn(t.ctypes.data, xs.ctypes.data, W, ys.ctypes.data, H, r0, nr, int(terrain), inp.ctypes.data, pre.ctypes.data,
       out.ctypes.data, st.ctypes.data)
    return (pre if terrain else None), out, st


def normalise(f, terrain, zfactor=0, mn=None, mx=None):
    """_perlin_numpy / _terrain_numpy after the field: NumPy's own arithmetic in the cell type."""
    T = f.dtype.type
    mn = f.min() if mn is None else T(mn)
    mx = f.max() if mx is None else T(mx)
    with np.errstate(invalid="ignore", divide="ignore"):
        d = (f - mn) / (mx - mn)
    if terrain:
        d[d < T(0.3)] = 0
        d *= T(zfactor)
    return d


# ----------------------------------------------------------------------------- golden cases
def perlin_cases(g):
    m, f, off = g["perlin_meta"], g["perlin_freq"], g["perlin_off"]
    for k in range(len(m)):
        h, w, f64, seed, raised = (int(v) for v in m[k])
        dt = np.float64 if f64 else np.float32
        out = None if raised else g["perlin_out"][off[k]:off[k + 1]].reshape(h, w).astype(dt)
        yield dict(h=h, w=w, dtype=dt, seed=seed, freq=(f[k, 0], f[k, 1]), raised=bool(raised), out=out,
                   name="perlin%d" % k)


def perlin_coords(c):
    return (np.linspace(0, c["freq"][0], c["w"], endpoint=False, dtype=np.float32),
            np.linspace(0, c["freq"][1], c["h"], endpoint=False, dtype=np.float32))


def terrain_cases(g):
    m, off = g["terrain_meta"], g["terrain_off"]
    for k in range(len(m)):
        h, w, f64, seed, zf, has_ext, nan_at = (int(v) for v in m[k])
        dt = np.float64 if f64 else np.float32
        data = np.full((h, w), g["terrain_fill"][k], dt)
        if nan_at >= 0:
            data.ravel()[nan_at] = np.nan
        r = g["terrain_ranges"][k]
        sl = slice(off[k], off[k + 1])
        yield dict(h=h, w=w, dtype=dt, seed=seed, zfactor=zf, data=data, x_range=(r[0], r[1]), y_range=(r[2], r[3]),
                   full_extent=tuple(g["terrain_extent"][k]) if has_ext else None, scaled=g["terrain_scaled"][k],
                   out=g["terrain_out"][sl].reshape(h, w).astype(dt), pre=g["terrain_precube"][sl].reshape(h, w).astype(dt),
                   name="terrain%d" % k)


def terrain_coords(c):
    s = c["scaled"]
    return (np.linspace(s[0], s[1], c["w"], endpoint=False, dtype=np.float32),
            np.linspace(s[2], s[3], c["h"], endpoint=False, dtype=np.float32))


def check_terrain_close(got, ref, zfactor, name):
    """Within the cube's rounding of the reference, and the water decision different only near the threshold."""
    assert got.dtype == ref.dtype and got.shape == ref.shape, name
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(got), nan), name
    tol = (F32_TOL if ref.dtype == np.float32 else F64_TOL) * abs(zfactor)
    g, r = got[~nan].astype(np.float64), ref[~nan].astype(np.float64)
    water = (g == 0) != (r == 0)
    assert np.all(np.abs(g - r)[~water] <= tol), (name, np.abs(g - r)[~water].max())
    near = np.abs(np.maximum(g, r)[water] / zfactor - 0.3) <= 2 * tol / abs(zfactor)
    assert near.all(), name


# ----------------------------------------------------------------------------- CPU: the header
def test_header_permutation_equals_numpy_at_2_20(host):
    for s in SEED_LIST:
        a, _, _, _ = host_perm(host, s, N)
        assert np.array_equal(a, np.random.RandomState(s).permutation(N)), s


@pytest.mark.parametrize("n", [1, 2, 3, 5, 31, 32, 33, 63, 64, 65, 100, 127, 128, 129, 1000, 1024, 1025, 4097,
                               65535, 65536, 65537])
def test_header_permutation_equals_numpy_at_small_n(host, n):
    for s in (0, 7, 2 ** 32 - 1):
        a, _, _, _ = host_perm(host, s, n)
        assert np.array_equal(a, np.random.RandomState(s).permutation(n)), (s, n)


@pytest.mark.parametrize("n", [2, 33, 64, 65, 96, 97, 129, 257, 1025, 2049, 4096, 4097, 65537, N])
def test_chunk_rule_equals_sequential_draws(host, n):
    # every power-of-two boundary below n is crossed, and the last 63 steps run at i < 64
    for s in (0, 5, 10, 2 ** 32 - 1):
        a0, j0, w0, _ = host_perm(host, s, n)
        a1, j1, w1, _ = host_perm(host, s, n, chunked=True)
        assert np.array_equal(j0[1:n], j1[1:n]), (s, n)
        assert w1 >= w0 and w1 - w0 < 32
        assert np.array_equal(a0, a1)


@pytest.mark.parametrize("n", [2, 3, 17, 100, 1000, 65537, N])
def test_reservation_rounds_equal_sequential_shuffle(host, n):
    for s in (0, 5, 2 ** 32 - 1):
        a0, _, _, _ = host_perm(host, s, n)
        a1, _, _, rounds = host_perm(host, s, n, chunked=True, reserved=True)
        assert np.array_equal(a0, a1), (s, n)
        assert 1 <= rounds < max(2, n)


def test_header_perlin_equals_reference(host, golden):
    mod = _mod("perlin")
    count = 0
    for c in perlin_cases(golden):
        xs, ys = perlin_coords(c)
        _, f, st = host_field(host, [c["seed"]], xs, ys, False, np.zeros((c["h"], c["w"]), c["dtype"]))
        assert mod.index_out_of_range(st) == c["raised"], c["name"]
        if c["raised"]:
            continue
        got = normalise(f, False)
        assert got.dtype == c["out"].dtype
        assert np.array_equal(got.view(np.uint8), c["out"].view(np.uint8), equal_nan=False) or \
            np.array_equal(got, c["out"], equal_nan=True), c["name"]
        count += 1
    assert count > 250


def test_header_terrain_equals_reference(host, golden):
    mod = _mod("perlin")
    for c in terrain_cases(golden):
        xs, ys = terrain_coords(c)
        seeds = list(range(c["seed"], c["seed"] + 16))
        pre, f, st = host_field(host, seeds, xs, ys, True, c["data"])
        assert not mod.index_out_of_range(st)
        assert np.array_equal(pre, c["pre"], equal_nan=True), c["name"]
        check_terrain_close(normalise(f, True, c["zfactor"]), c["out"], c["zfactor"], c["name"])
    nan = [c for c in terrain_cases(golden) if np.isnan(c["data"]).any()]
    assert nan and all(np.isnan(c["out"]).all() for c in nan)


def test_docstring_example(golden):
    want = np.array([[0.39268944, 0.27577767, 0.01621884, 0.05518942],
                     [1., 0.8229485, 0.2935367, 0.],
                     [1., 0.8715414, 0.41902685, 0.02916668]], np.float32)
    c = next(perlin_cases(golden))
    assert (c["h"], c["w"], c["seed"]) == (3, 4, 5)
    np.testing.assert_allclose(c["out"], want, rtol=1e-6)


# ----------------------------------------------------------------------------- CPU: arguments
class _Dask:
    __module__ = "dask.array.core"
    shape, ndim, dtype = (4, 4), 2, np.dtype(np.float32)


class _Agg:
    def __init__(self, data, dims=("y", "x"), attrs=None):
        self.data, self.dims, self.attrs = data, dims, attrs or {}
        self.shape = getattr(data, "shape", None)


def test_argument_errors_before_any_cuda_call():
    perlin, terrain = _mod("perlin").perlin, _mod("terrain").generate_terrain
    z = np.zeros((4, 5), np.float32)
    for bad in (-1, 2 ** 32, 2 ** 40):
        with pytest.raises(ValueError, match="Seed must be between"):
            perlin(_Agg(z), seed=bad)
    for bad in (-1, 2 ** 32 - 15, 2 ** 32 - 1):
        with pytest.raises(ValueError, match="Seed must be between"):
            terrain(_Agg(z), seed=bad)
    with pytest.raises(TypeError):
        perlin(_Agg(z), seed=1.5)
    assert _mod("perlin").check_seed(2 ** 32 - 16, 16)[-1] == 2 ** 32 - 1
    for dt in (np.int32, np.int16, np.uint8, np.float16, np.int64, np.complex64):
        for f in (perlin, terrain):
            with pytest.raises(TypeError):
                f(_Agg(np.zeros((4, 5), dt)))
    for shape in ((0, 5), (4, 0), (0, 0)):
        for f in (perlin, terrain):
            with pytest.raises(ValueError):
                f(_Agg(np.zeros(shape, np.float32)))
    for shape in ((4,), (2, 3, 4)):
        for f in (perlin, terrain):
            with pytest.raises(ValueError):
                f(_Agg(np.zeros(shape, np.float32)))
    for f in (perlin, terrain):
        with pytest.raises(NotImplementedError):
            f(_Agg(_Dask()))
        with pytest.raises(TypeError):
            f(_Agg([[0.0, 1.0]]))


def test_full_extent_keeps_the_reference_condition():
    terrain = _mod("terrain").generate_terrain
    z = _Agg(np.zeros((4, 5), np.float32))
    with pytest.raises(TypeError, match="tuple\\(4\\)"):
        terrain(z, full_extent=np.zeros(3))
    with pytest.raises(TypeError):
        terrain(z, full_extent=5)   # len() of an int
    with pytest.raises(IndexError):
        terrain(z, full_extent=(0, 0, 1))   # a tuple passes the check and is indexed at 3
    with pytest.raises(ZeroDivisionError):
        terrain(z, x_range=(3, 3))
    with pytest.raises(ZeroDivisionError):
        terrain(z, full_extent=(0, 2, 0, 5))


def test_scale_and_pixel_centres():
    t = _mod("terrain")
    assert t._scale(100, (0, 500), (0.0, 1.0)) == 0.2
    assert t._scale(-250, (0, 500), (0.0, 1.0)) == -0.5
    np.testing.assert_array_equal(t._pixel_centres((0, 500), 50), (np.arange(50) + 0.5) * 10)
    c = t._pixel_centres((-20e6, 20e6), 400)
    s = 400 / 40e6
    np.testing.assert_array_equal(c, (np.arange(400) + 0.5 - 20e6 * s) / s)
    assert np.all(np.diff(c) > 0)


def test_signatures_match_reference():
    with open(os.path.join(GOLDEN, "terrain_signature.json")) as f:
        want = json.load(f)
    import xrspatial_b200
    for mod, fn in (("perlin", "perlin"), ("terrain", "generate_terrain")):
        got = [[k, v.default] for k, v in inspect.signature(getattr(_mod(mod), fn)).parameters.items()]
        assert [k for k, _ in got] == [k for k, _ in want[fn]]
        for (k, d), (_, (kind, val)) in zip(got, want[fn]):
            if kind == "callable":
                assert d is inspect.Parameter.empty, k
            else:
                assert repr(d) == val, k
        assert getattr(xrspatial_b200, fn) is getattr(_mod(mod), fn)


def _lib():
    lib = importlib.import_module("xrspatial_b200._lib")
    try:
        lib.lib()
    except lib.XrsError:
        pytest.skip("libxrs_b200.so not built")
    return lib


def test_c_entry_points_check_arguments():
    L = _lib()
    P = ctypes.c_void_p
    fake = P(4096)   # never dereferenced: every call below fails its checks first
    n = ctypes.c_int64()
    seeds = (ctypes.c_uint32 * 2)(1, 2)

    def msg():
        return L.lib().xrs_last_error_string().decode()

    tb = L.lib().xrs_perm_tables_scratch_bytes
    assert tb(1, N, None) == L.XRS_EINVAL
    assert tb(0, N, ctypes.byref(n)) == L.XRS_EINVAL and "n_seeds" in msg()
    assert tb(33, N, ctypes.byref(n)) == L.XRS_EINVAL
    assert tb(1, N + 1, ctypes.byref(n)) == L.XRS_EINVAL and "2^20" in msg()
    assert tb(16, N, ctypes.byref(n)) == L.XRS_OK
    assert 16 * 20 * N <= n.value < 16 * 24 * N
    assert tb(2, 100, ctypes.byref(n)) == L.XRS_OK
    tables = L.lib().xrs_perm_tables
    assert tables(None, 2, 100, fake, fake, n.value, None, None) == L.XRS_EINVAL and "seed" in msg()
    assert tables(seeds, 2, 100, None, fake, n.value, None, None) == L.XRS_EINVAL and "tables" in msg()
    assert tables(seeds, 2, 100, fake, None, n.value, None, None) == L.XRS_EINVAL and "NULL scratch" in msg()
    assert tables(seeds, 2, 100, fake, fake, n.value - 1, None, None) == L.XRS_EINVAL and "too small" in msg()

    nb = L.lib().xrs_noise_scratch_bytes
    assert nb(0, 4, 0, ctypes.byref(n)) == L.XRS_EINVAL
    assert nb(4, 4, 0, None) == L.XRS_EINVAL
    assert nb(4, 10, 1, ctypes.byref(n)) == L.XRS_OK

    def noise(**kw):
        a = dict(inp=fake, dt=0, pitch=40, H=4, W=10, t=fake, xs=fake, ys=fake, terrain=1, out=fake, op=40,
                 st=fake, scr=fake, sb=n.value)
        a.update(kw)
        return L.lib().xrs_noise(a["inp"], a["dt"], a["pitch"], a["H"], a["W"], a["t"], a["xs"], a["ys"],
                                 a["terrain"], 4000.0, a["out"], a["op"], a["st"], a["scr"], a["sb"], None)

    assert noise(dt=2) == L.XRS_EINVAL and "float32 or float64" in msg()
    assert noise(inp=None) == L.XRS_EINVAL and "NULL input" in msg()
    assert noise(pitch=36) == L.XRS_EINVAL and "input pitch" in msg()
    assert noise(dt=1) == L.XRS_EINVAL and "input pitch" in msg()
    assert noise(op=44 + 2) == L.XRS_EINVAL and "output pitch" in msg()
    assert noise(out=None) == L.XRS_EINVAL and "NULL output" in msg()
    assert noise(t=None) == L.XRS_EINVAL and "NULL tables" in msg()
    assert noise(ys=None) == L.XRS_EINVAL
    assert noise(st=None) == L.XRS_EINVAL and "index_stats" in msg()
    assert noise(scr=None) == L.XRS_EINVAL and "NULL scratch" in msg()
    assert noise(sb=n.value - 1) == L.XRS_EINVAL and "too small" in msg()
    assert noise(H=0) == L.XRS_EINVAL


# ----------------------------------------------------------------------------- GPU
def _torch():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch


@pytest.mark.gpu
def test_device_tables_equal_numpy():
    _torch()
    mod = _mod("perlin")
    rounds = []
    t = mod.perm_tables(SEED_LIST, "cuda", rounds).cpu().numpy()
    for k, s in enumerate(SEED_LIST):
        assert np.array_equal(t[k], np.random.RandomState(s).permutation(N)), s
    assert 1 <= rounds[0] < 200


@pytest.mark.gpu
def test_device_tables_at_small_n():
    torch = _torch()
    L = _mod("_lib")
    for n in (1, 2, 33, 1000, 65537):
        seeds = [0, 5, 2 ** 32 - 1]
        need = ctypes.c_int64()
        L.call("xrs_perm_tables_scratch_bytes", len(seeds), n, ctypes.byref(need))
        t = torch.empty((len(seeds), n), dtype=torch.int32, device="cuda")
        scr = torch.empty(need.value, dtype=torch.uint8, device="cuda")
        L.call("xrs_perm_tables", ctypes.cast((ctypes.c_uint32 * 3)(*seeds), ctypes.c_void_p), 3, n,
               ctypes.c_void_p(t.data_ptr()), ctypes.c_void_p(scr.data_ptr()), need.value, None,
               ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        got = t.cpu().numpy()
        for k, s in enumerate(seeds):
            assert np.array_equal(got[k], np.random.RandomState(s).permutation(n)), (s, n)


def _agg(data, **kw):
    return _mod("_xr").DataArray(data, dims=("y", "x"), **kw)


def _bits_equal(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


@pytest.mark.gpu
def test_perlin_equals_every_golden(golden):
    torch = _torch()
    xb = _xb()
    for c in perlin_cases(golden):
        z = np.zeros((c["h"], c["w"]), c["dtype"])
        for data in (z, torch.from_numpy(z).cuda()):
            f = lambda: xb.perlin(_agg(data, attrs={"a": 1}), freq=c["freq"], seed=c["seed"])  # noqa: E731
            if c["raised"]:
                with pytest.raises(IndexError):
                    f()
                continue
            r = f()
            got = r.data if isinstance(r.data, np.ndarray) else r.data.cpu().numpy()
            assert _bits_equal(got, c["out"]) or np.array_equal(got, c["out"], equal_nan=True), c["name"]
            assert r.name == "perlin" and tuple(r.dims) == ("y", "x") and dict(r.attrs) == {"a": 1}
            assert type(r.data) is type(data)


def _xb():
    return importlib.import_module("xrspatial_b200")


@pytest.mark.gpu
def test_perlin_on_a_second_stream_and_a_row_offset_view(golden):
    torch = _torch()
    xb = _xb()
    c = [c for c in perlin_cases(golden) if (c["h"], c["w"]) == (37, 53) and not c["raised"]][5]
    buf = torch.full((c["h"] + 7, c["w"] + 11), 3.5, dtype=torch.float32 if c["dtype"] == np.float32
                     else torch.float64, device="cuda")
    view = buf[5:5 + c["h"], 2:2 + c["w"]]
    before = buf.clone()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        r = xb.perlin(_agg(view), freq=c["freq"], seed=c["seed"], name="n")
        got = r.data.cpu().numpy()
    s.synchronize()
    assert _bits_equal(got, c["out"]) and r.name == "n"
    assert torch.equal(buf, before)


@pytest.mark.gpu
def test_terrain_equals_host_restatement_and_golden(host, golden):
    torch = _torch()
    xb = _xb()
    for c in terrain_cases(golden):
        xs, ys = terrain_coords(c)
        _, f, _ = host_field(host, list(range(c["seed"], c["seed"] + 16)), xs, ys, True, c["data"])
        want = normalise(f, True, c["zfactor"])
        for data in (c["data"], torch.from_numpy(c["data"]).cuda()):
            before = np.array(c["data"], copy=True)
            r = xb.generate_terrain(_agg(data), x_range=c["x_range"], y_range=c["y_range"], seed=c["seed"],
                                    zfactor=c["zfactor"], full_extent=c["full_extent"])
            got = r.data if isinstance(r.data, np.ndarray) else r.data.cpu().numpy()
            assert _bits_equal(got, want) or np.array_equal(got, want, equal_nan=True), c["name"]
            check_terrain_close(got, c["out"], c["zfactor"], c["name"])
            host_in = data if isinstance(data, np.ndarray) else data.cpu().numpy()
            assert _bits_equal(host_in, before)
            if np.isnan(c["data"]).any():
                assert np.isnan(got).all()
            assert tuple(r.dims) == ("y", "x") and r.name == "terrain"
            xc = np.asarray(getattr(r.coords["x"], "data", r.coords["x"]))
            yc = np.asarray(getattr(r.coords["y"], "data", r.coords["y"]))
            np.testing.assert_array_equal(xc, _mod("terrain")._pixel_centres(c["x_range"], c["w"]))
            np.testing.assert_array_equal(yc, _mod("terrain")._pixel_centres(c["y_range"], c["h"]))
            rx = (c["x_range"][1] - c["x_range"][0]) / c["w"]
            ry = (c["y_range"][1] - c["y_range"][0]) / c["h"]
            np.testing.assert_allclose(r.attrs["res"], (rx, ry), rtol=1e-9)


def _raw_noise(torch, data, seeds, xs, ys, terrain, zfactor):
    """xrs_noise through the C ABI: the output and the field's min and max before normalisation."""
    mod, L = _mod("perlin"), _mod("_lib")
    H, W = data.shape
    tables = mod.perm_tables(seeds, data.device)
    dx = torch.from_numpy(np.asarray(xs, np.float32)).cuda()
    dy = torch.from_numpy(np.asarray(ys, np.float32)).cuda()
    need = ctypes.c_int64()
    L.call("xrs_noise_scratch_bytes", H, W, int(terrain), ctypes.byref(need))
    scr = torch.empty(need.value, dtype=torch.uint8, device="cuda")
    out = torch.empty_like(data)
    st = torch.empty((len(seeds), 5), dtype=torch.int32, device="cuda")
    esz = data.element_size()
    L.call("xrs_noise", ctypes.c_void_p(data.data_ptr()), 0 if data.dtype == torch.float32 else 1, W * esz, H, W,
           ctypes.c_void_p(tables.data_ptr()), ctypes.c_void_p(dx.data_ptr()), ctypes.c_void_p(dy.data_ptr()),
           int(terrain), float(zfactor), ctypes.c_void_p(out.data_ptr()), W * esz, ctypes.c_void_p(st.data_ptr()),
           ctypes.c_void_p(scr.data_ptr()), need.value, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    mm = scr[:16].cpu().numpy().view(np.float64)
    assert not mod.index_out_of_range(st.cpu().numpy())
    return out.cpu().numpy(), mm


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_full_field_and_its_extremes_equal_host_at_1024(host, dt):
    torch = _torch()
    n = 1024
    xs = np.linspace(0.0, 1.0, n, endpoint=False, dtype=np.float32)
    ys = np.linspace(-0.25, 0.75, n, endpoint=False, dtype=np.float32)
    data = torch.zeros((n, n), dtype=torch.float32 if dt == np.float32 else torch.float64, device="cuda")
    for terrain, seeds in ((False, [7]), (True, list(range(3, 19)))):
        got, mm = _raw_noise(torch, data, seeds, xs * (1 if terrain else 9), ys * (1 if terrain else 9), terrain, 10)
        _, f, _ = host_field(host, seeds, xs * (1 if terrain else 9), ys * (1 if terrain else 9), terrain,
                             np.zeros((n, n), dt))
        assert mm[0] == f.min() and mm[1] == f.max()
        assert _bits_equal(got, normalise(f, terrain, 10))


@pytest.mark.gpu
def test_8192_sampled_rows_equal_host(host):
    torch = _torch()
    n = 8192
    rows = [0, 1, 4095, 4096, 8191]
    xs = np.linspace(0.0, 1.0, n, endpoint=False, dtype=np.float32)
    data = torch.zeros((n, n), dtype=torch.float32, device="cuda")
    for terrain, seeds, scale in ((False, [5], 40.0), (True, list(range(10, 26)), 1.0)):
        got, (mn, mx) = _raw_noise(torch, data, seeds, xs * np.float32(scale), xs * np.float32(scale), terrain, 4000)
        for r in rows:
            _, f, _ = host_field(host, seeds, xs * np.float32(scale), xs * np.float32(scale), terrain, None, (r, 1))
            assert mn <= f.min() and f.max() <= mx
            assert _bits_equal(got[r:r + 1], normalise(f, terrain, 4000, mn, mx)), (terrain, r)


@pytest.mark.gpu
def test_repeated_calls_are_bit_identical():
    torch = _torch()
    xb = _xb()
    z = torch.zeros((700, 900), dtype=torch.float32, device="cuda")
    a = xb.generate_terrain(_agg(z)).data.cpu().numpy()
    b = xb.generate_terrain(_agg(z)).data.cpu().numpy()
    p = xb.perlin(_agg(z), freq=(13, 7)).data.cpu().numpy()
    q = xb.perlin(_agg(z), freq=(13, 7)).data.cpu().numpy()
    assert _bits_equal(a, b) and _bits_equal(p, q)


@pytest.mark.gpu
def test_one_cell_perlin_is_nan():
    _torch()
    r = _xb().perlin(_agg(np.zeros((1, 1), np.float64)))
    assert np.isnan(r.data).all() and r.data.dtype == np.float64

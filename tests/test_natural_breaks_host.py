"""natural_breaks without a GPU: MT19937 jump-ahead (mt19937.cuh compiled with g++) against NumPy's stream, the
chunked resolve and first[] chains of the device sample as a host model against NumPy's shuffle, a NumPy
statement of the Jenks column passes against the reference's matrices, the host backtrack and warnings against
every golden break, and the public signature."""
import ctypes
import inspect
import json
import os
import subprocess
import sys
import warnings

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
HEADER = os.path.join(ROOT, "xarray-spatial_b200", "csrc", "mt19937.cuh")
SEED = 1234567890


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(GOLDEN, "natural_breaks_reference.npz"), allow_pickle=False))


def numpy_sample(n, s, seed=SEED):
    idx = np.linspace(0, n, n, endpoint=False, dtype=np.uint32)
    np.random.RandomState(seed).shuffle(idx)
    return np.sort(idx[:s]).astype(np.int64)


# ----------------------------------------------------------------------------- the header on the host
@pytest.fixture(scope="module")
def host(tmp_path_factory):
    d = tmp_path_factory.mktemp("mt")
    cpp, so = str(d / "m.cpp"), str(d / "m.so")
    with open(cpp, "w") as f:
        f.write('#include "%s"\n' % HEADER + r"""
#include <algorithm>
using namespace xrs::mt;
static Poly g_phi;
static const Poly &phi() { if (g_phi.empty()) g_phi = mt_char_poly(); return g_phi; }
extern "C" int mt_phi_degree() { return phi().empty() ? -1 : kMtBits; }
// The 624 words from word d on (d a multiple of 624) of init_genrand(seed)'s stream, by jump-ahead.
extern "C" void mt_words_at(uint32_t seed, uint64_t d, uint32_t *out) {
    uint32_t s[kMtN], j[kMtN];
    mt_init(s, seed);
    mt_jump(s, poly_x_pow_mod(d, phi()), j);
    mt_twist(j);
    for (int i = 0; i < kMtN; ++i) out[i] = mt_temper(j[i]);
}
// The device sample's algorithm on the host: chunks of `chunk` words from jumped states (a doubling tree of
// jumps), the warp chunk rule of the resolve simulated lane by lane, counts from guessed first steps re-scanned
// until no start moves, first[] as max(n - i), the chains and the sorted set.  Returns the rounds taken.
static uint32_t resolve_chunk(const uint32_t *w, int64_t len, uint32_t i, uint32_t lo, int64_t n, uint32_t *first) {
    for (int64_t q = 0; q < len && i >= lo; q += 32) {
        bool fast = chunk_uniform(i);
        const uint32_t m = interval_mask(i);
        for (int l = 0; l < 32 && fast; ++l) fast = !undecided(w[q + l] & m, i);
        if (fast) {
            uint32_t acc = 0;
            for (int l = 0; l < 32; ++l) {
                const uint32_t v = w[q + l] & m;
                if (sure_accept(v, i)) {
                    const uint32_t step = i - acc;
                    if (first && step >= lo && v != step) first[v] = std::max(first[v], (uint32_t)(n - step));
                    ++acc;
                }
            }
            i -= acc;
        } else {
            for (int l = 0; l < 32 && i >= lo; ++l) {
                const uint32_t v = w[q + l] & interval_mask(i);
                if (v <= i) {
                    if (first && v != i) first[v] = std::max(first[v], (uint32_t)(n - i));
                    --i;
                }
            }
        }
    }
    return i;
}
extern "C" long long nb_sample_model(uint32_t seed, int64_t n, int64_t s, int64_t chunk, int64_t chunks,
                                     int64_t *out) {
    const int64_t lo = std::max<int64_t>(s, 1);
    std::vector<uint32_t> st((size_t)chunks * kMtN), words((size_t)chunks * chunk);
    mt_init(st.data(), seed);
    Poly p = poly_x_pow_mod((uint64_t)chunk, phi());
    for (int64_t half = 1; half < chunks; half *= 2) {
        for (int64_t c = half; c < std::min(2 * half, chunks); ++c) mt_jump(&st[(c - half) * kMtN], p, &st[c * kMtN]);
        p = poly_square_mod(p, phi());
    }
    for (int64_t c = 0; c < chunks; ++c) {
        uint32_t mt[kMtN];
        std::copy(&st[c * kMtN], &st[c * kMtN] + kMtN, mt);
        for (int64_t b = 0; b < chunk / kMtN; ++b) {
            mt_twist(mt);
            for (int k = 0; k < kMtN; ++k) words[c * chunk + b * kMtN + k] = mt_temper(mt[k]);
        }
    }
    std::vector<int64_t> starts(chunks), counts(chunks);
    for (int64_t c = 0; c < chunks; ++c) starts[c] = std::max<int64_t>(n - 1 - c * chunk / 2, lo - 1);   // a guess
    std::vector<char> dirty(chunks, 1);
    long long rounds = 0;
    for (bool changed = true; changed;) {
        ++rounds;
        for (int64_t c = 0; c < chunks; ++c) {
            if (!dirty[c]) continue;
            if (starts[c] < lo) { counts[c] = 0; continue; }
            const uint32_t e = resolve_chunk(&words[c * chunk], chunk, (uint32_t)starts[c], (uint32_t)lo, n, nullptr);
            counts[c] = starts[c] - std::max<int64_t>(e, lo - 1);
        }
        changed = false;
        int64_t carry = 0;
        for (int64_t c = 0; c < chunks; ++c) {
            const int64_t v = std::max<int64_t>(n - 1 - carry, lo - 1);
            dirty[c] = v != starts[c];
            changed |= dirty[c];
            starts[c] = v;
            carry += counts[c];
        }
        if (!changed && n - 1 - carry > lo - 1) return -1;   // the stream is too short
    }
    std::vector<uint32_t> first(n, 0);
    for (int64_t c = 0; c < chunks; ++c)
        if (starts[c] >= lo) resolve_chunk(&words[c * chunk], chunk, (uint32_t)starts[c], (uint32_t)lo, n, first.data());
    std::vector<char> mark(n, 0);
    for (int64_t q = 0; q < s; ++q) {
        int64_t x = q;
        while (first[x]) x = n - (int64_t)first[x];
        mark[x] = 1;
    }
    int64_t k = 0;
    for (int64_t x = 0; x < n; ++x) if (mark[x]) out[k++] = x;
    return rounds;
}
""")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, cpp])
    lib = ctypes.CDLL(so)
    lib.mt_words_at.argtypes = [ctypes.c_uint32, ctypes.c_uint64, ctypes.c_void_p]
    lib.mt_words_at.restype = None
    lib.nb_sample_model.argtypes = [ctypes.c_uint32, ctypes.c_int64, ctypes.c_int64, ctypes.c_int64, ctypes.c_int64,
                                    ctypes.c_void_p]
    lib.nb_sample_model.restype = ctypes.c_longlong
    return lib


def test_berlekamp_massey_finds_the_degree_19937_polynomial(host):
    assert host.mt_phi_degree() == 19937


def test_jumped_states_continue_numpys_stream(host):
    """The state d words ahead, by x^d mod phi and Horner, yields NumPy's words d .. d + 623, d past 2^32 too."""
    bg = np.random.RandomState(SEED)._bit_generator
    at = 0
    offsets = [0, 624, 624 * 832, 624 * 832 * 5 + 624 * 7, 624 * 6883000]   # the last is past 2^32 words
    assert offsets[-1] > 2 ** 32
    for d in offsets:
        while at < d:
            step = min(d - at, 1 << 24)
            bg.random_raw(step)
            at += step
        want = bg.random_raw(624).astype(np.uint32)
        at += 624
        got = np.zeros(624, np.uint32)
        host.mt_words_at(SEED, d, got.ctypes.data)
        assert np.array_equal(got, want), d


@pytest.mark.parametrize("n", [2, 3, 1023, 1024, 1025, 65535, 65536, 65537, 2 ** 20 + 1, 2000003])
def test_chunked_resolve_and_chains_give_numpys_sample(host, n):
    chunk = 624 * 64   # many chunks, so the speculated starts really move
    for s in sorted({1, 2, 8, 1000, 20000, n // 2, n - 1}):
        if not 1 <= s < n:
            continue
        need = 1.5 * n + 16 * np.sqrt(n) + 4 * chunk
        chunks = int(need // chunk) + 1
        out = np.zeros(s, np.int64)
        rounds = host.nb_sample_model(SEED, n, s, chunk, chunks, out.ctypes.data)
        assert rounds > 0, (n, s)
        assert np.array_equal(out, numpy_sample(n, s)), (n, s)


# ----------------------------------------------------------------------------- the Jenks column passes
def jenks_columns(x, k):
    """_run_numpy_jenks_matrices restated column by column: pass j fills column j of every row at once, each row
    running its m-loop in the reference's order -- float64 sums of float32 values and float32 squares, the
    variance with an IEEE divide, float32 storage, ties to the later m."""
    x = np.asarray(x, np.float32)
    n = x.size
    lcl = np.zeros((n + 1, k + 1), np.float32)
    var = np.zeros((n + 1, k + 1), np.float32)
    lcl[1, 1:] = 1.0
    var[2:, 1:] = np.inf
    if n < 2:
        return lcl, var
    rows = np.arange(2, n + 1)
    for j in range(1, k + 1):
        s = np.zeros(n - 1)
        ss = np.zeros(n - 1)
        best = var[2:, j].copy()
        lim = lcl[2:, j].copy()
        final = np.zeros(n - 1)
        for m in range(n):
            a = max(0, m - 1)
            i4 = rows[a:] - m - 1
            val = x[i4]
            s[a:] += val.astype(np.float64)
            ss[a:] += (val * val).astype(np.float64)
            variance = ss[a:] - (s[a:] * s[a:]) / (m + 1.0)
            if j == 1:
                if m >= 1:
                    final[m - 1] = variance[0]
                continue
            nv = variance + var[i4, j - 1].astype(np.float64)
            upd = (best[a:].astype(np.float64) >= nv) & (i4 != 0)
            idx = np.nonzero(upd)[0] + a
            lim[idx] = (rows[idx] - m).astype(np.float32)
            best[idx] = nv[upd].astype(np.float32)
        if j == 1:
            lcl[2:, 1] = 1.0
            var[2:, 1] = final.astype(np.float32)
        else:
            lcl[2:, j], var[2:, j] = lim, best
    return lcl, var


def test_column_passes_match_the_reference_matrices(golden):
    tags = [k[len("jenks_data__"):] for k in golden if k.startswith("jenks_data__")]
    assert len(tags) >= 5
    for tag in tags:
        data = golden["jenks_data__" + tag]
        k = golden["jenks_lcl__" + tag].shape[1] - 1
        lcl, var = jenks_columns(data.astype(np.float32), k)
        assert np.array_equal(lcl.view(np.uint32), golden["jenks_lcl__" + tag].view(np.uint32)), tag
        assert np.array_equal(var.view(np.uint32), golden["jenks_var__" + tag].view(np.uint32)), tag


# ----------------------------------------------------------------------------- the host side, every golden break
def golden_calls(g):
    return json.loads(str(g["calls"]))


def host_bins(cl, raster, kw, cache):
    """natural_breaks_bins' host steps over a NumPy sample and the NumPy column passes: (bins, uvk, warnings)."""
    num_sample, k = kw.get("num_sample", 20000), kw.get("k", 5)
    msgs = []
    flat = raster.ravel()
    fin = flat[np.isfinite(flat)]
    if fin.size == 0:
        raise ValueError("all-NaN")
    max_data = float(np.max(fin))
    n = flat.size
    if num_sample is not None and num_sample < n:
        size = len(range(n)[:num_sample])
        sample = flat[numpy_sample(n, size)] if size > 0 else flat[:0]
    else:
        sample = flat
    if sample.size >= 40000:
        msgs.append("O(n^2)")
    data = np.sort(sample[np.isfinite(sample)])
    uv = np.unique(data)
    if uv.size < k:
        return uv, uv.size, msgs + ["Not enough unique values"]
    if data.size > 1100:
        return None, uv.size, msgs   # the GPU tests take the larger samples
    key = (id(raster), num_sample if num_sample is None or num_sample < n else None)
    if key not in cache or cache[key].shape[1] < k + 1:
        cache[key] = jenks_columns(data.astype(np.float32), max(k, 10))[0]
    return cl.jenks_backtrack(data, cache[key][:, :k + 1], k, max_data), uv.size, msgs


def test_host_backtrack_and_warnings_reproduce_every_golden_break(golden):
    sys.path.insert(0, ROOT)
    from xrspatial_b200 import classify as cl
    cache, cases, checked = {}, {}, 0
    for case, kw, tag in golden_calls(golden):
        if "gen__" + case in golden or "bad" in tag:
            continue
        raster = cases.setdefault(case, golden["case__" + case])
        if "err__" + tag in golden:
            with pytest.raises(Exception) as e:
                host_bins(cl, raster, kw, cache)
            assert str(golden["err__" + tag]) == "ValueError" and e.type is ValueError
            continue
        bins, uvk, msgs = host_bins(cl, raster, kw, cache)
        if bins is None:
            continue
        want = golden["bins__" + tag]
        assert bins.dtype == want.dtype and np.array_equal(bins, want), tag
        assert np.array_equal(np.arange(uvk), golden["newv__" + tag]), tag
        gw = [str(m) for m in golden.get("warn__" + tag, [])]
        assert len(gw) == len(msgs) and all(w in g for w, g in zip(msgs, gw)), tag
        checked += 1
    assert checked >= 30


def test_signature_matches_the_reference():
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    from make_golden import encode_default
    from xrspatial_b200 import classify as cl
    import xrspatial_b200
    ref = json.load(open(os.path.join(GOLDEN, "natural_breaks_signature.json")))
    for fn in (cl.natural_breaks, xrspatial_b200.natural_breaks):
        got = [[k, encode_default(v.default)] for k, v in inspect.signature(inspect.unwrap(fn)).parameters.items()]
        assert got == ref["natural_breaks"]


def test_warning_texts_are_the_references(golden):
    """The texts natural_breaks warns with, formatted as the reference formats them."""
    sys.path.insert(0, ROOT)
    from xrspatial_b200 import classify as cl
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        cl._warn("x")
    assert caught[0].category is Warning
    assert str(golden["warn__big_ns50000_k7"][0]).startswith("natural_breaks Warning: Natural break")

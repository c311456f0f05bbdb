"""Shared test helpers: tolerances of the parity gate (SURVEY.md section 8d), input makers, and the harness of
the tests that call the C entry points on the GPU directly."""
import ctypes

import numpy as np

# what xrs_debug_last_used_tma reports (LaunchKind in csrc/common.cuh)
(K_STRIP_CPASYNC, K_STRIP_TMA, K_INGEST, K_BOX, K_CONV_TILED, K_CONV_DIRECT, K_FUSED, K_STAT_TILED, K_STAT_DIRECT,
 K_ZONAL, K_ZONAL_PAIR) = range(11)

SENTINEL = 0x5A


def gpu_lib():
    """The loaded library module (xrspatial_b200._lib); fails when no CUDA device is present."""
    import torch
    import xrspatial_b200
    assert torch.cuda.is_available(), "these tests need a CUDA device"
    return xrspatial_b200._lib


def stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def last_kind(lib):
    return lib.lib().xrs_debug_last_used_tma()


def raster(H, W, seed, nan_frac=0.01):
    """A float32 random-walk surface around 500 with `nan_frac` of its cells NaN."""
    rng = np.random.default_rng(seed)
    z = rng.standard_normal((H, W)).cumsum(0).cumsum(1) * 3.0 + 500.0
    z[rng.random((H, W)) < nan_frac] = np.nan
    return z.astype(np.float32)


def in_buffer(z, pad_cols=0, rows_above=0, rows_below=0, shift=0):
    """z on the device inside a larger buffer: `pad_cols` extra cells per row (pitch), `rows_above` /
    `rows_below` extra rows of other data (a row-offset view), `shift` cells past the 16-byte aligned start
    (shift=1: base and pitch not 16-byte aligned, so no TMA).  The extra cells hold large finite values, so a
    kernel that reads them gives a visibly wrong answer.  Returns (tensor, pointer, pitch in bytes); keep the
    tensor referenced while kernels read it."""
    import torch
    H, W = z.shape
    big = np.full((H + rows_above + rows_below, W + pad_cols + shift), 9.0e3, dtype=z.dtype)
    big[rows_above:rows_above + H, shift:shift + W] = z
    t = torch.from_numpy(big).cuda()
    isz = t.element_size()
    return t, t.data_ptr() + (rows_above * t.stride(0) + shift) * isz, t.stride(0) * isz


class Pitched(object):
    """An output rectangle of H x W cells of `itemsize` bytes inside a sentinel-filled buffer: one row above and
    below, 4 cells left and 8 right, so the pitch stays a multiple of 16 bytes."""

    def __init__(self, H, W, itemsize=4):
        import torch
        self.H, self.W, self.isz = H, W, itemsize
        self.wp = W + 12
        self.buf = torch.full(((H + 2) * self.wp * itemsize,), SENTINEL, dtype=torch.uint8, device="cuda")
        self.ptr = self.buf.data_ptr() + (self.wp + 4) * itemsize
        self.pitch = self.wp * itemsize

    def inside(self, what):
        """The bytes of the H x W rectangle, as an (H, W * itemsize) uint8 array, after checking that no byte
        outside it changed."""
        b = self.buf.cpu().numpy().reshape(self.H + 2, self.pitch)
        lo, hi = 4 * self.isz, (4 + self.W) * self.isz
        ins = b[1:1 + self.H, lo:hi].copy()
        b[1:1 + self.H, lo:hi] = SENTINEL
        bad = int((b != SENTINEL).sum())
        assert bad == 0, "%s: %d bytes outside the raster were written" % (what, bad)
        return ins


def assert_same_nan(a, b, what=""):
    np.testing.assert_array_equal(np.isnan(a), np.isnan(b), err_msg="NaN mask differs " + what)


def assert_close_f32(gpu, ref, rtol=1e-5, atol=1e-6, what=""):
    """|gpu - ref| <= rtol*|ref| + atol, identical NaN masks (float32 ops, bar 1e-5 relative)."""
    gpu = np.asarray(gpu, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    assert gpu.shape == ref.shape, (gpu.shape, ref.shape)
    assert_same_nan(gpu, ref, what)
    m = ~np.isnan(ref)
    inf = m & np.isinf(ref)
    np.testing.assert_array_equal(gpu[inf], ref[inf])
    m &= ~np.isinf(ref)
    err = np.abs(gpu[m] - ref[m])
    tol = rtol * np.abs(ref[m]) + atol
    bad = err > tol
    assert not bad.any(), "%s: %d cells out of tolerance, worst err %g (ref %g)" % (
        what, bad.sum(), err[bad].max(), ref[m][bad][np.argmax(err[bad])])


def assert_aspect_close(gpu, ref, what=""):
    """aspect: -1 (flat) mask identical, NaN mask identical, circular distance within
    1e-5 relative + 1e-4 degrees."""
    gpu = np.asarray(gpu, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    assert_same_nan(gpu, ref, what)
    np.testing.assert_array_equal(gpu == -1, ref == -1, err_msg="flat mask differs " + what)
    m = ~np.isnan(ref) & (ref != -1)
    d = np.abs(gpu[m] - ref[m])
    d = np.minimum(d, 360.0 - d)
    tol = 1e-5 * np.abs(ref[m]) + 1e-4
    assert (d <= tol).all(), "%s: aspect worst circular err %g" % (what, d.max())


def terrain(rng, h, w, water=False, nans=0.0, integer=False, zmax=4000.0):
    z = rng.standard_normal((h, w)).cumsum(0).cumsum(1)
    z += np.linspace(0, 30, w)[None, :] + np.linspace(0, 10, h)[:, None]
    z = (z - z.min()) / (z.max() - z.min() + 1e-9) * zmax
    if water:
        z[z < 0.3 * z.max()] = 0.0
    if integer:
        z = np.round(z)
    z = z.astype(np.float32)
    if nans:
        z[rng.random((h, w)) < nans] = np.nan
    return z


def box_magnitude_fields(rng, H, W):
    """Quantised fields on which ordinary window sums are exact or nearly so: terrain at multiples of 1/256 in
    [0, 4096], the same with a 1e6 offset, and a lognormal field over 1e-2 .. 1e6 rounded to 8 significant
    bits."""
    t = rng.standard_normal((H, W)).cumsum(0).cumsum(1)
    t = (t - t.min()) / max(t.max() - t.min(), 1e-9) * 4096.0
    terr = (np.round(t * 256.0) / 256.0).astype(np.float32)
    m, e = np.frexp(np.exp(rng.uniform(np.log(1e-2), np.log(1e6), (H, W))))
    logn = np.ldexp(np.round(m * 256.0) / 256.0, e).astype(np.float32)
    return {"terrain": terr, "offset": (terr.astype(np.float64) + 1e6).astype(np.float32), "lognormal": logn}


def box_planted_values(M):
    """Cells far beyond data whose largest |x| is M: 2^24 M, 1e15 .. 1e29 (1e20 is the CMIP fill value), the
    float32 below 2^100, 2^100 and FLT_MAX."""
    return [np.float32(M * 2.0 ** 24), np.float32(1e15), np.float32(1e20), np.float32(1e25), np.float32(1e29),
            np.nextafter(np.float32(2.0 ** 100), np.float32(0)), np.float32(2.0 ** 100),
            np.float32(3.4028235e38)]


def box_window_errors(got, ref, planted, kh, kw, w, M, what):
    """Windows without NaN / inf / planted cells: |got - ref| <= 2 ulp32(ref) + 2^-36 |w| kh kw M (pass w = 1 for
    a mean).  Windows holding one: the same NaN mask and rtol 1e-6.  Returns the worst clean |got - ref|
    relative to the window scale |w| kh kw M."""
    from scipy.ndimage import maximum_filter
    touched = maximum_filter(planted.astype(np.uint8), size=(kh, kw), mode="constant", cval=0) > 0
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref), err_msg=what + ": NaN masks differ")
    clean = ~touched & np.isfinite(ref)
    scale = abs(w) * kh * kw * M
    err = np.abs(got[clean].astype(np.float64) - ref[clean].astype(np.float64))
    bound = 2.0 * np.spacing(np.abs(ref[clean])).astype(np.float64) + 2.0 ** -36 * scale
    bad = err > bound
    assert not bad.any(), "%s: %d clean windows off by up to %.3g (%.3g of the window scale)" % (
        what, int(bad.sum()), err.max(), err.max() / scale)
    odd = touched & ~np.isnan(ref)
    np.testing.assert_allclose(got[odd], ref[odd], rtol=1e-6, err_msg=what + ": windows with planted cells")
    return float(err.max() / scale) if err.size else 0.0


def box_plant(z, value, rows, rng):
    """`value` planted at the given rows, alternating signs, every third one as a 3-row vertical run; returns
    the raster and the mask of planted cells."""
    H, W = z.shape
    z = z.copy()
    mask = np.zeros(z.shape, bool)
    for i, y in enumerate(sorted(set(r for r in rows if 0 <= r < H))):
        x = int(rng.integers(0, W))
        for dy in range(3 if i % 3 == 0 else 1):
            if y + dy < H:
                z[y + dy, x] = value if i % 2 else -value
                mask[y + dy, x] = True
    return z, mask

"""binary, reclassify, quantile, percentiles, box_plot, equal_interval, std_mean, head_tail_breaks,
maximum_breaks and natural_breaks (classify.py of the reference) on the GPU, following the reference's NumPy path.

Every scheme ends in one per-cell pass: the reference's binary-search bin lookup (`_cpu_bin`) or the membership
test of `binary` (`_cpu_binary`).  The breaks come from device work on the raster -- exact order statistics
(radix select), one moments pass per level, or a radix sort -- and from the reference's own host arithmetic on
the few scalars that work returns, restated line for line, so that they are NumPy's breaks bit for bit.  std_mean
and head_tail_breaks take their means and deviations from float64 sums instead of NumPy's float32 pairwise ones
(DESIGN.md section 4.11).

natural_breaks draws the reference's seeded sample of cell indices on the device (RandomState(1234567890)'s shuffle,
without the shuffle: xrs_nb_sample), sorts the sampled cells there, fills its Jenks matrices column by column on
the device, bit for bit, and runs the reference's backtrack over them on the host.
"""
import ctypes
import warnings

import numpy as np

from . import _lib
from ._xr import DataArray
from .dataset_support import supports_dataset
from .proximity import _cells
from .utils import is_dask_array, is_device_array, like_container, stream_ptr

CELLS, GAPS, TIE_POSITIONS = 0, 1, 2    # key sources of xrs_classify_select
_KEY_BITS = {np.dtype(np.float64): 64, np.dtype(np.int64): 64, np.dtype(np.int16): 16, np.dtype(np.uint16): 16}


def _key_dtype(dtype):
    return np.uint64 if _KEY_BITS.get(dtype, 32) == 64 else np.uint32


def _values(keys, dtype):
    """The cells of `dtype` whose order-preserving keys (xrs_b200.h, classify) are `keys`."""
    kt = _key_dtype(dtype)
    k = np.asarray(keys, dtype=np.uint64).astype(kt)
    if dtype.kind == "f":
        top = kt(1) << kt(8 * kt().itemsize - 1)
        return np.where(k & top, k & ~top, ~k).astype(kt).view(dtype)
    bits = 8 * dtype.itemsize
    if dtype.kind == "i":
        k = k ^ kt(1 << (bits - 1))
    return k.astype(np.dtype("u%d" % dtype.itemsize)).view(dtype)


class _Raster:
    """The raster on the device in a cell type the kernels read, and what the reference's arithmetic needs to
    know about it: `dtype`, the numpy type of its cells before widening."""

    def __init__(self, agg):
        import torch
        data = agg.data
        if is_dask_array(data):
            raise NotImplementedError("classify: Dask arrays are not supported by the GPU backend")
        if not (isinstance(data, np.ndarray) or is_device_array(data)):
            raise TypeError("Unsupported Array Type: {}".format(type(data)))
        self.data = data
        self.t, self.code = _cells(data)
        self.cells = np.dtype(str(self.t.dtype).replace("torch.", ""))
        if isinstance(data, np.ndarray):
            self.dtype = data.dtype
        else:
            src = str(getattr(data, "dtype", self.t.dtype)).replace("torch.", "")
            self.dtype = np.dtype(src) if src not in ("bfloat16",) else self.cells
        self.torch = torch
        self._hist0 = self._n = None

    def call(self, name, *args):
        with self.torch.cuda.device(self.t.device):
            _lib.call(name, *args, stream_ptr(self.t))

    def _ptr(self):
        return ctypes.c_void_p(self.t.data_ptr())

    def _pitch(self):
        return self.t.stride(0) * self.t.element_size() if self.t.dim() == 2 else 0

    def scratch(self, query, *args):
        need = ctypes.c_int64()
        _lib.call(query, *args, ctypes.byref(need))
        return self.torch.empty(max(1, need.value), dtype=self.torch.uint8, device=self.t.device), need.value

    # ------------------------------------------------------------------ device work
    def cells_pass(self, member, table, new_values=None):
        torch = self.torch
        H, W = self.t.shape
        out = torch.empty((H, W), dtype=self.t.dtype if member else torch.float32, device=self.t.device)
        tab = np.ascontiguousarray(np.asarray(table, dtype=np.float64).ravel())
        nb = tab.size
        dev_tab = torch.as_tensor(np.append(tab, 0.0), device=self.t.device)
        dev_new = None
        if not member:
            nv = np.asarray(new_values).astype(np.float32).ravel()[:nb]
            # The reference reads past the end of new_values for a bin without one (quantile, when
            # np.arange's steps give one percentile more than k): NaN, no class, here.
            nv = np.append(nv, np.full(nb + 1 - nv.size, np.nan, np.float32))
            dev_new = torch.as_tensor(nv, device=self.t.device)
        if H and W:
            self.call("xrs_classify_cells", self._ptr(), self.code, self._pitch(), H, W, int(member),
                      ctypes.c_void_p(dev_tab.data_ptr()),
                      None if dev_new is None else ctypes.c_void_p(dev_new.data_ptr()), nb,
                      ctypes.c_void_p(out.data_ptr()), out.stride(0) * out.element_size())
        return out

    def moments(self, above=-np.inf):
        """(count, mean, M2, min, max) of the finite cells above `above`, in float64."""
        H, W = self.t.shape
        scratch, size = self.scratch("xrs_classify_moments_scratch_bytes")
        out = self.torch.empty(5, dtype=self.torch.float64, device=self.t.device)
        self.call("xrs_classify_moments", self._ptr(), self.code, self._pitch(), H, W, float(above),
                  ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(scratch.data_ptr()), size)
        n, mean, m2, mn, mx = out.cpu().numpy().tolist()
        return int(n), mean, m2, mn, mx

    def _select(self, source, ptr, H, W, bits, ranks, hist0, tie=0):
        scratch, size = self.scratch("xrs_classify_select_scratch_bytes")
        ranks = np.ascontiguousarray(ranks, dtype=np.int64)
        nr = ranks.size
        keys = np.zeros(max(1, nr), np.uint64)
        rem = np.zeros(max(1, nr), np.int64)
        n = ctypes.c_int64()
        self.call("xrs_classify_select", source, ptr, self.code, self._pitch() if source == CELLS else 0, H, W,
                  bits, ctypes.c_uint64(tie), ranks.ctypes.data_as(ctypes.c_void_p), nr,
                  keys.ctypes.data_as(ctypes.c_void_p), rem.ctypes.data_as(ctypes.c_void_p), ctypes.byref(n),
                  hist0.ctypes.data_as(ctypes.c_void_p), ctypes.c_void_p(scratch.data_ptr()), size)
        return n.value, keys[:nr], rem[:nr]

    def finite_count(self):
        if self._n is None:
            self._hist0 = np.zeros(256, np.uint64)
            H, W = self.t.shape
            self._n = self._select(CELLS, self._ptr(), H, W, _KEY_BITS.get(self.cells, 32), [], self._hist0)[0]
        return self._n

    def order_stats(self, ranks):
        """The finite cells at 0-based `ranks` of their ascending order, as `dtype`: one set of digit passes."""
        self.finite_count()
        H, W = self.t.shape
        _, keys, _ = self._select(CELLS, self._ptr(), H, W, _KEY_BITS.get(self.cells, 32), ranks, self._hist0)
        return _values(keys, self.cells).astype(self.dtype)

    def sorted_keys(self):
        """The finite cells' keys, sorted on the device, and their number."""
        torch = self.torch
        H, W = self.t.shape
        kt = _key_dtype(self.cells)
        keys = torch.empty(max(1, H * W), dtype=torch.int64 if kt == np.uint64 else torch.int32,
                           device=self.t.device)
        scratch, size = self.scratch("xrs_classify_sort_scratch_bytes", H * W, self.code)
        n = ctypes.c_int64()
        self.call("xrs_classify_sort", self._ptr(), self.code, self._pitch(), H, W, ctypes.c_void_p(keys.data_ptr()),
                  ctypes.byref(n), ctypes.c_void_p(scratch.data_ptr()), size)
        return keys, n.value

    def with_cells(self, t):
        """The same cell type over other device cells `t` (2-D)."""
        other = object.__new__(_Raster)
        other.__dict__.update(self.__dict__)
        other.t, other._hist0, other._n = t, None, None
        return other

    def sorted_values(self):
        """The finite cells, sorted, on the host in the cells' own type: what the reference's data.sort() gives."""
        keys, n = self.sorted_keys()
        host = keys[:n].cpu().numpy().view(_key_dtype(self.cells))
        return _values(host, self.cells).astype(self.dtype)

    def max_break_stats(self):
        gaps = _SortedGaps(self)
        if self.cells != self.dtype and self.dtype.itemsize <= 2:
            # bool / int8 / uint8 / float16 cells were widened, and np.diff in their own type wraps or rounds
            # where the wider one does not; they have at most 65536 unique values, so the gaps are taken from those
            return _UniqueGaps(gaps.unique_values())
        return gaps


class _SortedGaps:
    """What maximum_breaks reads of np.unique(finite cells) and its np.diff, from the device-sorted keys."""

    def __init__(self, r):
        self.r = r
        self.keys, self.n = r.sorted_keys()
        self.ptr = ctypes.c_void_p(self.keys.data_ptr())
        self.bits = _KEY_BITS.get(r.cells, 32)
        self.hist0 = np.zeros(256, np.uint64)
        self.n_gaps = r._select(GAPS, self.ptr, 1, self.n, self.bits, [], self.hist0)[0] if self.n else 0

    def unique_count(self):
        return self.n_gaps + 1 if self.n else 0

    def _host_keys(self, k):
        return k.cpu().numpy().view(_key_dtype(self.r.cells))

    def _pick(self, mode, cap, tie=0, pos=0):
        torch = self.r.torch
        out = torch.empty(max(1, cap * (1 + mode)), dtype=self.keys.dtype, device=self.keys.device)
        scratch = torch.empty(8, dtype=torch.uint8, device=self.keys.device)
        count = ctypes.c_int64()
        self.r.call("xrs_classify_pick", self.ptr, self.r.code, self.n, mode, ctypes.c_uint64(tie), pos,
                    ctypes.c_void_p(out.data_ptr()), cap, ctypes.byref(count), ctypes.c_void_p(scratch.data_ptr()))
        if count.value != cap:
            raise _lib.XrsError("classify pick found %d entries, expected %d" % (count.value, cap))
        return self._host_keys(out[:cap * (1 + mode)])

    def unique_values(self):
        u = self.unique_count()
        return np.sort(_values(self._pick(0, u) if u else np.zeros(0), self.r.cells).astype(self.r.dtype))

    def largest(self):
        return _values(self._host_keys(self.keys[self.n - 1:self.n]), self.r.cells).astype(self.r.dtype)[0]

    def gap_pairs(self, start):
        """(uv[i], uv[i + 1]) for the gaps at ranks start .. of np.argsort(np.diff(uv), kind='stable'), in the
        order of i."""
        tie, pos = 0, 0
        if start > 0:
            _, key, rem = self.r._select(GAPS, self.ptr, 1, self.n, self.bits, [start], self.hist0)
            tie = int(key[0])
            pbits = max(8, -(-int(self.n - 1).bit_length() // 8) * 8)
            h = np.zeros(256, np.uint64)
            self.r._select(TIE_POSITIONS, self.ptr, 1, self.n, pbits, [], h, tie)
            _, p, _ = self.r._select(TIE_POSITIONS, self.ptr, 1, self.n, pbits, [int(rem[0])], h, tie)
            pos = int(p[0])
        pairs = self._pick(1, self.n_gaps - start, tie, pos).reshape(-1, 2)
        pairs = pairs[np.argsort(pairs[:, 0], kind="stable")]
        v = _values(pairs.ravel(), self.r.cells).astype(self.r.dtype).reshape(-1, 2)
        return v[:, 0], v[:, 1]


class _UniqueGaps:
    """The same reads over the sorted unique values themselves, np.diff taken in their own type."""

    def __init__(self, uv):
        self.uv = uv

    def unique_count(self):
        return self.uv.size

    def unique_values(self):
        return self.uv

    def largest(self):
        return self.uv[-1]

    def gap_pairs(self, start):
        idx = np.sort(np.argsort(np.diff(self.uv), kind="stable")[start:])
        return self.uv[idx], self.uv[idx + 1]


# ---------------------------------------------------------------------- the reference's host arithmetic
def _quantile_is_valid(q):
    if q.ndim == 1 and q.size < 10:
        for i in range(q.size):
            if not (0.0 <= q[i] <= 1.0):
                return False
    elif not (q.min() >= 0 and q.max() <= 1):
        return False
    return True


def _lerp(a, b, t):
    diff_b_a = np.subtract(b, a)
    lerp_interpolation = np.asanyarray(np.add(a, diff_b_a * t))
    np.subtract(b, diff_b_a * (1 - t), out=lerp_interpolation, where=t >= 0.5, casting="unsafe",
                dtype=type(lerp_interpolation.dtype))
    if lerp_interpolation.ndim == 0:
        lerp_interpolation = lerp_interpolation[()]
    return lerp_interpolation


def _percentile_plan(n, dtype, q):
    """np.percentile(a, q) of n values of `dtype` (method 'linear'), up to fetching values: the virtual indexes,
    the previous / next indexes (-1 the last) and gamma, in NumPy's dtypes."""
    q = np.true_divide(q, dtype.type(100) if dtype.kind == "f" else 100, out=...)
    if not _quantile_is_valid(q):
        raise ValueError("Percentiles must be in the range [0, 100]")
    if q.ndim > 2:
        raise ValueError("q must be a scalar or 1d")
    virtual = np.asanyarray((n - 1) * q)
    prev = np.asanyarray(np.floor(virtual))
    nxt = np.asanyarray(prev + 1)
    above = virtual >= n - 1
    if above.any():
        prev[above] = -1
        nxt[above] = -1
    below = virtual < 0
    if below.any():
        prev[below] = 0
        nxt[below] = 0
    if np.issubdtype(dtype, np.inexact):
        nans = np.isnan(virtual)
        if nans.any():
            prev[nans] = -1
            nxt[nans] = -1
    prev = prev.astype(np.intp)
    nxt = nxt.astype(np.intp)
    gamma = np.asanyarray(np.asanyarray(virtual - prev), dtype=virtual.dtype).reshape(virtual.shape)
    return prev, nxt, gamma


def percentiles_of(stats, dtype, qs, largest=False):
    """[np.percentile(finite values, q) for q in qs], the finite values being `stats`' (n of them, fetched by
    rank), as `dtype`, then the largest finite value when `largest`: every rank in one order-statistics call."""
    n = stats.finite_count()
    if n == 0:
        return [np.percentile(np.empty(0, dtype), q) for q in qs]   # raises as the reference does
    plans = [_percentile_plan(n, dtype, q) for q in qs]
    ranks = np.unique(np.concatenate([np.concatenate((p.ravel(), x.ravel())) % n for p, x, _ in plans]
                                     + [np.array([n - 1])]))
    vals = np.asarray(stats.order_stats(ranks)).astype(dtype)
    out = []
    for prev, nxt, gamma in plans:
        a = vals[np.searchsorted(ranks, prev % n)]
        b = vals[np.searchsorted(ranks, nxt % n)]
        out.append(_lerp(a, b, gamma))
    if largest:
        out.append(vals[-1])
    return out


def quantile_bins(stats, k):
    """classify.py:396-405 `_run_quantile`, numpy module."""
    w = 100.0 / k
    p = np.arange(w, 100 + w, w)
    if p[-1] > 100.0:
        p[-1] = 100.0
    q = percentiles_of(stats, stats.dtype, [p])[0]
    return np.unique(q)


def percentiles_bins(stats, pct):
    """classify.py:1110-1180: the unique percentiles and the largest finite value."""
    q, max_v = percentiles_of(stats, stats.dtype, [pct], largest=True)
    q_np = np.asarray(np.unique(q))
    max_v = float(max_v)
    return np.sort(np.unique(np.append(q_np, max_v)))


def box_plot_bins(stats, hinge):
    """classify.py:1286-1315 `_run_box_plot`, numpy module: its finite data went through np.where(isinf, nan),
    so integer cells are float64 there."""
    dtype = stats.dtype if stats.dtype.kind == "f" else np.dtype(np.float64)
    q1, q2, q3, max_v = (float(v) for v in percentiles_of(stats, dtype, [25, 50, 75], largest=True))
    iqr = q3 - q1
    raw_bins = [q1 - hinge * iqr, q1, q2, q3, q3 + hinge * iqr, max_v]
    bins = np.sort(np.unique(raw_bins))
    bins = bins[bins <= max_v]
    if bins[-1] < max_v:
        bins = np.append(bins, max_v)
    return bins


def equal_interval_bins(stats, k):
    """classify.py:837-866 `_run_equal_interval`, numpy module; returns (cuts, number of new values)."""
    n, _, _, mn, mx = stats.moments()
    min_data = float(mn) if n else np.nan
    max_data = float(mx) if n else np.nan
    width = (max_data - min_data) / k
    cuts = np.arange(min_data + width, max_data + width, width)
    l_cuts = cuts.shape[0]
    if l_cuts > k:
        cuts = cuts[0:k]
    cuts[-1] = max_data
    return cuts, l_cuts


def _result_type(dtype):
    """The dtype of np.nanmean / np.nanstd over the reference's cleaned data: the cells' own float type, else
    float64."""
    return dtype if dtype.kind == "f" else np.dtype(np.float64)


def std_mean_bins(stats):
    """classify.py:943-967 `_run_std_mean` with the mean and standard deviation from float64 moments, rounded
    to the type NumPy returns them in."""
    n, mean, m2, _, mx = stats.moments()
    rt = _result_type(stats.dtype).type
    if n:
        mean_v, std_v, max_v = float(rt(mean)), float(rt(np.sqrt(m2 / n))), float(mx)
    else:
        mean_v = std_v = max_v = np.nan
    return np.sort(np.unique([mean_v - 2 * std_v, mean_v - std_v, mean_v + std_v, mean_v + 2 * std_v, max_v]))


def head_tail_bins(stats):
    """classify.py:1013-1027 `_compute_head_tail_bins`: one moments pass over the cells above each mean."""
    n, mean, _, _, mx = stats.moments()
    if n == 0:
        np.nanmax(np.empty(0, stats.dtype))   # raises as the reference does
    rt = _result_type(stats.dtype).type
    bins = []
    count, m = n, mean
    while count > 1:
        mean_v = float(rt(m))
        bins.append(mean_v)
        head, head_mean = stats.moments(mean_v)[:2]
        if head == 0 or head / count > 0.40:
            break
        count, m = head, head_mean
    if not bins:
        bins = [float(rt(mean))]
    bins.append(float(mx))
    return np.array(bins)


def maximum_breaks_bins(gaps, k):
    """classify.py:1191-1202 `_compute_maximum_break_bins` over the device's sorted unique values."""
    n_u = gaps.unique_count()
    if n_u < k:
        return gaps.unique_values()
    if n_u == 0:
        raise IndexError("index -1 is out of bounds for axis 0 with size 0")
    n_g = n_u - 1
    n_gaps = min(k - 1, n_g)
    start = slice(-n_gaps, None).indices(n_g)[0]    # np.argsort(diffs, kind='stable')[-n_gaps:]
    lo, hi = gaps.gap_pairs(start)
    bins = (lo + hi) / 2.0
    return np.append(bins, float(gaps.largest()))


NB_SEED = 1234567890     # the reference's RandomState seed for natural_breaks' sample


def _warn(message):
    with warnings.catch_warnings():
        warnings.simplefilter('default')
        warnings.warn(message, Warning, stacklevel=4)


def sample_indices(n, s, device, seed=NB_SEED):
    """np.sort(idx[:s]) for idx = np.linspace(0, n, n, dtype=uint32) after RandomState(seed).shuffle(idx), on the
    device as int64 (1 <= s < n <= 2^32)."""
    import torch
    need = ctypes.c_int64()
    _lib.call("xrs_nb_sample_scratch_bytes", n, s, ctypes.byref(need))
    scratch = torch.empty(need.value, dtype=torch.uint8, device=device)
    out = torch.empty(s, dtype=torch.int64, device=device)
    rounds = ctypes.c_int64()
    with torch.cuda.device(device):
        _lib.call("xrs_nb_sample", n, s, ctypes.c_uint32(seed), ctypes.c_void_p(out.data_ptr()),
                  ctypes.c_void_p(scratch.data_ptr()), need.value, ctypes.byref(rounds),
                  ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream))
    return out


def jenks_matrices(x, k):
    """_run_numpy_jenks_matrices over the sorted float32 DEVICE values x: (lower_class_limits, var_combinations)
    as DEVICE float32 tensors of shape (k + 1, n + 1), the transpose of the reference's."""
    import torch
    n = x.numel()
    need = ctypes.c_int64()
    _lib.call("xrs_nb_jenks_scratch_bytes", n, k, ctypes.byref(need))
    scratch = torch.empty(need.value // 4, dtype=torch.float32, device=x.device)
    lcl = torch.empty((k + 1, n + 1), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        _lib.call("xrs_nb_jenks", ctypes.c_void_p(x.data_ptr()), n, k, ctypes.c_void_p(lcl.data_ptr()),
                  ctypes.c_void_p(scratch.data_ptr()), need.value,
                  ctypes.c_void_p(torch.cuda.current_stream(x.device).cuda_stream))
    return lcl, scratch[:(k + 1) * (n + 1)].view(k + 1, n + 1)


def jenks_backtrack(data, lower_class_limits, n_classes, max_data):
    """classify.py `_run_jenks` after the matrices, and `bins = centroids[1:]; bins[-1] = max_data`: data is the
    sorted sample, lower_class_limits the (n + 1) x (k + 1) matrix."""
    k = data.shape[0]
    kclass = np.zeros(n_classes + 1, dtype=np.float32)
    kclass[0] = data[0]
    kclass[-1] = data[-1]
    count_num = n_classes
    while count_num > 1:
        elt = int(lower_class_limits[k][count_num] - 2)
        kclass[count_num - 1] = data[elt]
        k = int(lower_class_limits[k][count_num] - 1)
        count_num -= 1
    bins = np.array(kclass[1:])
    bins[-1] = max_data
    return bins


def natural_breaks_bins(r, num_sample, k):
    """classify.py:589-664 `_compute_natural_break_bins` with `max_data` (classify.py:737-743): (bins, uvk)."""
    n_finite, _, _, _, mx = r.moments()
    if n_finite == 0:
        np.max(np.empty(0, r.dtype))   # raises as the reference does
    max_data = float(mx)
    H, W = r.t.shape
    num_data = H * W
    sample = r
    size = num_data
    if num_sample is not None and num_sample < num_data:
        size = len(range(num_data)[:num_sample])   # idx[:num_sample]: negative sizes count from the end
        if size > 0:
            idx = sample_indices(num_data, size, r.t.device)
            # torch gathers unsigned 16- to 64-bit cells only through their signed view of the same width
            signed = {r.torch.uint16: r.torch.int16, r.torch.uint32: r.torch.int32, r.torch.uint64: r.torch.int64}
            t = r.t.view(signed[r.t.dtype]) if r.t.dtype in signed else r.t
            sample = r.with_cells(t[idx // W, idx % W].view(r.t.dtype).view(1, size))
        else:
            sample = r.with_cells(r.t.new_empty((1, 0)))
    if size >= 40000:
        _warn('natural_breaks Warning: Natural break '
              'classification (Jenks) has a complexity of O(n^2), '
              'your classification with {} data points may take '
              'a long time.'.format(size))
    data = sample.sorted_values()
    uvk = int(np.count_nonzero(data[1:] != data[:-1])) + 1 if data.size else 0
    if uvk < k:
        _warn('natural_breaks Warning: Not enough unique values '
              'in data array for {} classes. '
              'n_samples={} should be >= n_clusters={}. '
              'Using k={} instead.'.format(k, uvk, k, uvk))
        keep = np.ones(data.size, bool)
        keep[1:] = data[1:] != data[:-1]
        return data[keep], uvk
    if not isinstance(k, (int, np.integer)):
        raise TypeError("natural_breaks: k must be an integer, not {!r}".format(k))   # numba's typing error there
    if k < -1:
        raise ValueError("negative dimensions not allowed")   # np.zeros((n + 1, k + 1)) in the matrices
    if k < 1:
        raise IndexError("index -1 is out of bounds for axis 0 with size 0")   # kclass is too short
    lcl = np.zeros((data.size + 1, k + 1), np.float32)
    if k > 1:
        import torch
        x = torch.as_tensor(data.astype(np.float32), device=r.t.device)
        lcl = jenks_matrices(x, k)[0].cpu().numpy().T
    return jenks_backtrack(data, lcl, k, max_data), uvk


# ---------------------------------------------------------------------- public functions
def _bin(r, bins, new_values):
    return r.cells_pass(False, bins, new_values)


def _wrap(out, r, agg, name):
    if isinstance(out, np.ndarray):
        pass
    elif isinstance(r.data, np.ndarray):
        out = out.cpu().numpy()
    else:
        out = like_container(out, r.data)
    return DataArray(out, name=name, dims=agg.dims, coords=agg.coords, attrs=agg.attrs)


@supports_dataset
def binary(agg, values, name='binary'):
    """1 where a cell equals one of `values` (compared in float64), 0 where it is another finite value, NaN
    elsewhere (classify.py:87-149).  The output has the input's cell type."""
    r = _Raster(agg)
    out = r.cells_pass(True, np.asarray(values).astype(np.float64).ravel())
    if isinstance(r.data, np.ndarray):
        out = out.cpu().numpy().astype(r.dtype, copy=False)     # widened cells go back to their own type
    elif out.dtype != getattr(r.data, "dtype", out.dtype) and isinstance(r.data, r.torch.Tensor):
        out = out.to(r.data.dtype)
    return _wrap(out, r, agg, name)


@supports_dataset
def reclassify(agg, bins, new_values, name='reclassify'):
    """new_values[i] for the cells in bin i of `bins` by the reference's binary search (classify.py:273-393);
    NaN for non-finite cells and cells above the last bin.  float32."""
    if len(bins) != len(new_values):
        raise ValueError('bins and new_values mismatch. Should have same length.')
    r = _Raster(agg)
    return _wrap(_bin(r, bins, new_values), r, agg, name)


@supports_dataset
def quantile(agg, k=4, name='quantile'):
    """Classes of equal size from the exact percentiles of the finite cells (classify.py:426-505)."""
    r = _Raster(agg)
    q = quantile_bins(r, k)
    k_q = q.shape[0]
    if k_q < k:
        print("Quantile Warning: Not enough unique values"
              "for k classes (using {} bins)".format(k_q))
        k = k_q
    return _wrap(_bin(r, q, np.arange(k)), r, agg, name)


@supports_dataset
def percentiles(agg, pct=None, name='percentiles'):
    """Classes bounded by the percentiles `pct` (default [1, 10, 50, 90, 99]) of the finite cells and their
    maximum (classify.py:1121-1188)."""
    if pct is None:
        pct = [1, 10, 50, 90, 99]
    r = _Raster(agg)
    bins = percentiles_bins(r, pct)
    return _wrap(_bin(r, bins, np.arange(len(bins))), r, agg, name)


@supports_dataset
def box_plot(agg, hinge=1.5, name='box_plot'):
    """Classes bounded by the whiskers q1 - hinge IQR and q3 + hinge IQR, the quartiles and the maximum
    (classify.py:1343-1386)."""
    r = _Raster(agg)
    bins = box_plot_bins(r, hinge)
    return _wrap(_bin(r, bins, np.arange(len(bins))), r, agg, name)


@supports_dataset
def equal_interval(agg, k=5, name='equal_interval'):
    """k classes of equal width between the finite minimum and maximum (classify.py:870-940)."""
    r = _Raster(agg)
    cuts, l_cuts = equal_interval_bins(r, k)
    return _wrap(_bin(r, cuts, np.arange(l_cuts)), r, agg, name)


@supports_dataset
def std_mean(agg, name='std_mean'):
    """Classes bounded by the mean +- 1 and 2 standard deviations of the finite cells and their maximum
    (classify.py:971-1010)."""
    r = _Raster(agg)
    bins = std_mean_bins(r)
    return _wrap(_bin(r, bins, np.arange(len(bins))), r, agg, name)


@supports_dataset
def head_tail_breaks(agg, name='head_tail_breaks'):
    """Head/tail breaks: the mean of the values above the previous mean while the head holds at most 40 % of
    them, then the maximum (classify.py:1066-1107)."""
    r = _Raster(agg)
    bins = head_tail_bins(r)
    return _wrap(_bin(r, bins, np.arange(len(bins))), r, agg, name)


@supports_dataset
def maximum_breaks(agg, k=5, name='maximum_breaks'):
    """Breaks at the midpoints of the k - 1 widest gaps between the sorted unique finite values, then the
    maximum (classify.py:1240-1283)."""
    r = _Raster(agg)
    bins = maximum_breaks_bins(r.max_break_stats(), k)
    return _wrap(_bin(r, bins, np.arange(len(bins))), r, agg, name)


@supports_dataset
def natural_breaks(agg, num_sample=20000, name='natural_breaks', k=5):
    """Jenks natural breaks: the k classes of least within-class variance of a seeded sample of `num_sample` cells
    (every cell when None or not less than the cell count), bounded above by the finite maximum
    (classify.py:737-834).  The sample is the reference's; rasters of more than 2^32 cells raise ValueError."""
    r = _Raster(agg)
    bins, uvk = natural_breaks_bins(r, num_sample, k)
    return _wrap(_bin(r, bins, np.arange(uvk)), r, agg, name)

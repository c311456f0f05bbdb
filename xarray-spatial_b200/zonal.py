"""xrspatial.zonal.stats on the CUDA backend (reference: zonal.py:422-667).

One streaming pass (xrs_zonal_hash_run) discovers the zone ids and produces per-zone count /
sum / sum-of-squares / min / max partials; mean, std (ddof=0) and var are finalised from them in
float64.  `majority` counts (zone, value) pairs in a second pass (hash table; a device sort when
the values are too varied for the table).  Custom callables (`stats_funcs` given as a dict, exactly
like the reference: zonal.py:640-642) run per zone on the zone's valid values, grouped on the device
by one sort.  With `comm` (a torch.distributed process group) the partials of row-striped rasters
are combined with AllReduce before finalisation.
"""
import math

import numpy as np
import pandas as pd

from . import _lib
from ._xr import DataArray, Dataset
from .utils import (ArrayTypeFunctionMapping, as_device_tensor, call_on, device_cells, device_scratch, like_container,
                    pitch, ptr, to_container, validate_arrays)

_DEFAULT_STATS = ("mean", "max", "min", "sum", "std", "var", "count", "majority")


def _device_tensor(a):
    """A numpy array copied to the current CUDA device; a device array viewed as a torch tensor."""
    import torch
    if isinstance(a, np.ndarray):
        return torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return as_device_tensor(a)


def _prepare_zones(t):
    """Zone ids as the contiguous int32, int64, float32 or float64 tensor the kernels read: narrower integers and
    bool widen to int32, wider unsigned integers to int64, other floating types to float32."""
    import torch
    if t.dtype in (torch.int32, torch.int64, torch.float32, torch.float64):
        return t.contiguous()
    if t.dtype.is_floating_point:
        return t.to(torch.float32).contiguous()
    if t.dtype in (torch.int8, torch.int16, torch.uint8, torch.bool):
        return t.to(torch.int32).contiguous()
    return t.to(torch.int64).contiguous()


def _prepare_values(t):
    """Values as the contiguous float32 or float64 tensor the kernels read: float32 and float64 as they are, other
    floating types as float32, integers and bool as float64."""
    import torch
    if t.dtype in (torch.float32, torch.float64):
        return t.contiguous()
    return t.to(torch.float32 if t.dtype.is_floating_point else torch.float64).contiguous()


def _select_zones(present, zone_ids, keep_order=False):
    """(ids, pos): the zones a call reports and their positions in `present`, the sorted ids of the zones found in
    the raster.  Without `zone_ids`, every present zone, and `pos` is a slice, so that indexing with it copies
    nothing.  Otherwise the listed ids that are present: sorted and unique (zonal.stats), or in the caller's order
    with repeats kept when `keep_order` (crosstab).  `z in ndarray` compares with ==, so a NaN id never matches."""
    if zone_ids is None:
        return present, slice(None)
    listed = zone_ids if keep_order else np.unique(zone_ids)
    ids = np.array([z for z in listed if z in present], dtype=present.dtype)
    return ids, np.searchsorted(present, ids)


_EMPTY_KEY = -(1 << 63)


def _sample_pivot(values_t, comm=None):
    """One global shift p keeps sum((v-p)^2) well conditioned; the median of a small strided sample
    is enough (one tiny device-to-host copy), and unlike the mean it ignores huge nodata sentinels."""
    import torch
    flat = values_t.reshape(-1)
    step = max(1, flat.numel() // 4096)
    sample = flat[::step][:4096].to(torch.float64).cpu().numpy()
    sample = sample[np.isfinite(sample)]
    p0 = float(np.sort(sample)[sample.size // 2]) if sample.size else 0.0   # the device kernel's median
    if comm is not None:
        import torch.distributed as dist
        pt = torch.tensor([p0], dtype=torch.float64, device=values_t.device)
        dist.broadcast(pt, src=dist.get_global_rank(comm, 0), group=comm)
        p0 = float(pt.item())
    return p0


_MAX_OUT = 4096     # zones returned by the one-copy fast path of hash_partials
_HDR = 4            # header doubles of the packed result: used slots, overflow, pivot, INT64_MIN zone met


def _sentinel_partials(zones_t, values_t, nodata_values, pivot):
    """Partials of the zone INT64_MIN, which the device table cannot hold (its key is the table's empty
    key; the kernel only reports that it met the zone), by masked reductions over the raster."""
    import torch
    v = values_t.reshape(-1)
    ok = (zones_t.reshape(-1) == -(1 << 63)) & torch.isfinite(v)
    if nodata_values is not None:
        ok &= v != nodata_values
    vv = v[ok]
    d = vv.to(torch.float64) - pivot
    n = int(vv.numel())
    return dict(count=np.array([n], np.int64), s1=np.array([float(d.sum())]), s2=np.array([float((d * d).sum())]),
                min=np.array([float(vv.min()) if n else np.inf]), max=np.array([float(vv.max()) if n else -np.inf]))


def _empty_partials(nz):
    return dict(count=np.zeros(nz, np.int64), s1=np.zeros(nz), s2=np.zeros(nz), min=np.full(nz, np.inf),
                max=np.full(nz, -np.inf))


def _table_pass(entry, zones_t, values_t, nodata_values, table_args, keys, acc, sentinel_pivot=None):
    """One pass of the group-by entry point `entry` over the hash table `keys`, accumulating into `acc` (rows count
    as int64 bit patterns, s1, s2, min, max); `table_args` are the arguments between `nodata` and `count`, tensors
    passed by pointer.  None when the table overflowed, else (ids, part, pivot): the zones met, in table order;
    their partials; the shift of the sums.  The zone INT64_MIN, which the table cannot hold, is appended from
    masked reductions about `sentinel_pivot` (default: the pass's pivot)."""
    import torch
    dt = lambda t: _lib.DTYPES[str(t.dtype).replace("torch.", "")]  # noqa: E731
    packed = torch.empty(_HDR + 6 * _MAX_OUT, dtype=torch.float64, device=values_t.device)
    flags = torch.empty(3, dtype=torch.int32, device=values_t.device)
    call_on(values_t, entry, ptr(values_t), dt(values_t), ptr(zones_t), dt(zones_t), values_t.numel(),
            int(values_t.shape[-1]) if values_t.dim() else 1,
            0 if nodata_values is None else 1, 0.0 if nodata_values is None else float(nodata_values),
            *(ptr(a) if torch.is_tensor(a) else a for a in table_args), *(ptr(r) for r in acc),
            keys.numel(), ptr(packed), _MAX_OUT, ptr(flags))
    host = packed.cpu().numpy()                    # the one synchronising copy
    n_used, overflow, pivot, sentinel = int(host[0]), int(host[1]), float(host[2]), int(host[3])
    if overflow:
        return None
    if n_used <= _MAX_OUT:
        rows = host[_HDR:].reshape(6, _MAX_OUT)[:, :n_used]
    else:                                          # many zones: gather the used slots of the table itself
        used = torch.nonzero(keys != _EMPTY_KEY).reshape(-1)
        rows = torch.cat([keys[used].view(torch.float64)[None], acc[:, used]]).cpu().numpy()
    ids = _keys_to_ids(np.ascontiguousarray(rows[0]).view(np.int64), zones_t.dtype)
    part = dict(count=np.ascontiguousarray(rows[1]).view(np.int64).copy(), s1=rows[2].copy(), s2=rows[3].copy(),
                min=rows[4].copy(), max=rows[5].copy())
    if sentinel:
        ids = np.append(ids, np.int64(_EMPTY_KEY))
        sp = _sentinel_partials(zones_t, values_t, nodata_values, pivot if sentinel_pivot is None else sentinel_pivot)
        part = {n: np.append(a, sp[n]) for n, a in part.items()}
    return ids, part, pivot


def hash_partials(zones_t, values_t, nodata_values=None, comm=None, cap=1 << 16, table=None):
    """One streaming pass that discovers the zone ids and accumulates their partials
    (xrs_zonal_hash_run: pivot sampling, table init, accumulation and compaction are enqueued
    back to back; ONE device-to-host copy -- a 4-double header + 6 x 4096 doubles -- is the only
    synchronisation).  Returns (ids, part, pivot): ids = sorted unique finite zone values present
    in the raster (numpy, in the zones dtype), part = dict of numpy arrays aligned with ids
    (count int64; s1, s2, min, max float64), pivot = the scalar shift of s1/s2.
    With `comm`, the tables of all ranks are merged by id (and share one pivot).
    `table`: a dict that receives the device-side hash table (keys, cap) for `second_pass_partials`."""
    import torch
    dev = values_t.device
    hint = _sample_pivot(values_t, comm) if comm is not None else None
    if values_t.numel() == 0:
        return _keys_to_ids(np.zeros(0, np.int64), zones_t.dtype), _empty_partials(0), 0.0
    while True:
        # one blob: rows = keys, count (int64 bit patterns), s1, s2, min, max
        blob = torch.empty((6, cap), dtype=torch.float64, device=dev)
        keys = blob[0].view(torch.int64)
        res = _table_pass("xrs_zonal_hash_run", zones_t, values_t, nodata_values,
                          (0 if hint is None else 1, 0.0 if hint is None else float(hint), keys), keys, blob[1:])
        if res is not None:
            break
        if cap >= (1 << 24):
            raise NotImplementedError("more than 16M distinct zones are not supported")
        cap *= 16
    ids, part, pivot = res
    if table is not None:
        table.update(keys=keys, cap=cap)
    if comm is not None:
        ids, part = allreduce_tables(ids, part, dev, comm)
    order = np.argsort(ids, kind="stable")
    return ids[order], {n: a[order] for n, a in part.items()}, pivot


def _keys_to_ids(k, zones_dtype):
    """int64 table keys -> zone ids in the zones' dtype (float zones: the key is the float64 bit pattern)"""
    import torch
    if zones_dtype.is_floating_point:
        return k.view(np.float64).astype(np.float32 if zones_dtype == torch.float32 else np.float64)
    return k.astype(np.int32 if zones_dtype == torch.int32 else np.int64)


def second_pass_partials(zones_t, values_t, table, ids, means, nodata_values=None, comm=None):
    """numpy's two-pass variance: a second streaming pass over the hash table
    `hash_partials(..., table=...)` left on the device, with the sums taken about every zone's own
    mean (xrs_zonal_hash_second_pass; the means are scattered to the table's slots on the device, no
    host round trip beyond the one the first pass needed).  `ids`: sorted zone ids (numpy), `means`:
    float64, aligned -- over row stripes the merged ids / global means.  Returns the partials
    (count, s1, s2, min, max about `means`) aligned with `ids`."""
    import torch
    dev = values_t.device
    nz = len(ids)
    part = _empty_partials(nz)
    if nz and values_t.numel():
        keys, cap = table["keys"], table["cap"]
        fz = zones_t.dtype.is_floating_point
        ids_t = torch.as_tensor(np.asarray(ids, dtype=np.float64 if fz else np.int64), device=dev)
        means_t = torch.as_tensor(np.asarray(means, dtype=np.float64), device=dev)
        slot_ids = keys.view(torch.float64) if fz else keys
        idx = torch.searchsorted(ids_t, slot_ids).clamp_(max=nz - 1)
        pivots = means_t[idx].contiguous()                 # empty slots get some zone's mean: never read
        acc = torch.empty((5, cap), dtype=torch.float64, device=dev)
        # sorted ids: the INT64_MIN zone, when present, comes first
        local, lpart, _ = _table_pass("xrs_zonal_hash_second_pass", zones_t, values_t, nodata_values, (keys, pivots),
                                      keys, acc, sentinel_pivot=float(means[0]))
        pos = np.searchsorted(ids, local)
        for n in part:
            part[n][pos] = lpart[n]
    if comm is not None and nz:
        part = _allreduce_partials(part, dev, comm)
    return part


# the pair key's value half is the float32 bit pattern XOR this (csrc/zonal_hash.cu kZpValueXor): the
# table's empty key then stands for (zone INT32_MIN, a NaN), a pair that is never counted
_PAIR_VALUE_XOR = 0x7FC00000


class _PairTableOverflow(Exception):
    """more distinct (zone, value) pairs than the hash table is allowed to grow to"""


_PAIR_CAP = 1 << 20               # first size of the pair table
_PAIR_MAX_CAP = 1 << 26           # crosstab lets it grow to this (1 GiB of keys and counts)
_MAJORITY_PAIR_MAX_CAP = 1 << 24  # majority grows it no further and groups by one device sort instead


def _float32_exact(values_t):
    """`values_t` as float32, or None when a finite value is not exact in float32.  float32 rasters are used in
    place: the pair kernel itself folds -0.0 into 0.0, and a `+ 0.0` copy cost a full read + write of the raster."""
    import torch
    if values_t.dtype == torch.float32:
        return values_t
    vf = values_t.to(torch.float32)
    return vf if bool(((vf.to(values_t.dtype) == values_t) | ~torch.isfinite(values_t)).all()) else None


def _pair_inputs(zones_t, values_t):
    """The int32 zones and float32 values of the (zone, value) pair table; NotImplementedError when the
    narrowing would not be exact.  Cells whose float zone id is not finite get NaN values, so they drop out."""
    import torch
    zi = zones_t if zones_t.dtype == torch.int32 else zones_t.to(torch.int32)
    if zones_t.dtype.is_floating_point:
        finite_zone = torch.isfinite(zones_t)
        if not bool((zi.to(zones_t.dtype) == zones_t)[finite_zone].all()):
            raise NotImplementedError("'majority' needs integer-valued zone ids")
    elif zi is not zones_t and not bool((zi.to(zones_t.dtype) == zones_t).all()):
        raise NotImplementedError("'majority' needs zone ids that fit in int32")
    vf = _float32_exact(values_t)
    if vf is None:
        raise NotImplementedError("'majority' needs values that are exact in float32")
    if zones_t.dtype.is_floating_point:
        vf = torch.where(finite_zone, vf, torch.full_like(vf, float("nan")))
    return zi, vf


def pair_counts(zones_t, values_t, nodata_values=None, comm=None, cap=None, max_cap=None):
    """(zone ids int64, values float64, counts int64) of every distinct valid (zone, value) pair:
    one pass of xrs_zonal_pair_count over int32 zones and float32 values.  The table starts at `cap` slots
    (default _PAIR_CAP) and grows up to `max_cap` (default _PAIR_MAX_CAP), then raises _PairTableOverflow."""
    import torch
    if zones_t.dtype != torch.int32 or values_t.dtype != torch.float32:
        raise TypeError("pair_counts takes int32 zones and float32 values")
    cap = _PAIR_CAP if cap is None else cap
    max_cap = _PAIR_MAX_CAP if max_cap is None else max_cap
    dev = values_t.device
    vf, zi = values_t.contiguous(), zones_t.contiguous()
    while True:
        keys = torch.empty(cap, dtype=torch.int64, device=dev)
        count = torch.empty(cap, dtype=torch.int64, device=dev)
        ovf = torch.empty(1, dtype=torch.int32, device=dev)
        call_on(vf, "xrs_zonal_pair_count", ptr(vf), ptr(zi), vf.numel(), int(vf.shape[-1]) if vf.dim() else 1,
                0 if nodata_values is None else 1, 0.0 if nodata_values is None else float(nodata_values),
                ptr(keys), ptr(count), cap, ptr(ovf))
        if int(ovf.item()) == 0:
            break
        if cap >= max_cap:
            raise _PairTableOverflow()
        cap = min(cap * 16, max_cap)
    used = torch.nonzero(keys != _EMPTY_KEY).reshape(-1)
    k = keys[used].cpu().numpy()
    c = count[used].cpu().numpy()
    if comm is not None:
        import torch.distributed as dist
        gathered = [None] * dist.get_world_size(comm)
        dist.all_gather_object(gathered, (k, c), group=comm)
        k = np.concatenate([g[0] for g in gathered])
        c = np.concatenate([g[1] for g in gathered])
        k, inv = np.unique(k, return_inverse=True)
        c = np.bincount(inv, weights=c).astype(np.int64)
    zone = (k >> 32).astype(np.int64)
    val = ((k & 0xFFFFFFFF) ^ _PAIR_VALUE_XOR).astype(np.uint32).view(np.float32).astype(np.float64)
    return zone, val, c


def _total_order_bits(v32):
    """float32 tensor -> int64 keys in [0, 2^32) whose integer order is the float order."""
    import torch
    bits = v32.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    return torch.where(bits >= 0x80000000, 0xFFFFFFFF - bits, bits + 0x80000000)


def _majority_by_sort(zidx, vals, n_zones):
    """Majority per zone by one device sort.  zidx: int64 zone index per valid cell (0..n_zones-1),
    vals: the cells' values (float32: keyed by their order-preserving bit pattern; float64: keyed by
    their rank among the distinct values).  Returns a float64 numpy array of length n_zones (NaN for
    zones without cells): the most frequent value, smallest on ties (zonal.py:56-68)."""
    import torch
    out = np.full(n_zones, np.nan)
    if zidx.numel() == 0:
        return out
    if vals.dtype == torch.float32:
        vkey, table = _total_order_bits(vals), None
        span = 1 << 32
    else:
        table, vkey = torch.unique(vals, return_inverse=True)   # sorted distinct values, ranks
        span = int(table.numel())
    keys = zidx * span + vkey
    del vkey
    keys = torch.sort(keys).values
    uniq, cnt = torch.unique_consecutive(keys, return_counts=True)
    del keys
    zone = torch.div(uniq, span, rounding_mode="floor")
    zid, zinv = torch.unique_consecutive(zone, return_inverse=True)
    best = torch.zeros(zid.numel(), dtype=cnt.dtype, device=cnt.device).scatter_reduce_(0, zinv, cnt, "amax")
    pos = torch.arange(uniq.numel(), device=uniq.device)
    pos = torch.where(cnt == best[zinv], pos, torch.full_like(pos, uniq.numel()))
    first = torch.full((zid.numel(),), uniq.numel(), dtype=pos.dtype, device=pos.device).scatter_reduce_(0, zinv, pos, "amin")
    vk = uniq[first] - zid * span
    if table is None:
        b = torch.where(vk >= 0x80000000, vk - 0x80000000, 0xFFFFFFFF - vk)
        win = b.cpu().numpy().astype(np.uint32).view(np.float32).astype(np.float64)
    else:
        win = table[vk].to(torch.float64).cpu().numpy()
    out[zid.cpu().numpy()] = win
    return out


def majority_by_zone(zones_t, values_t, unique_zones, nodata_values=None, comm=None):
    """float64 numpy array aligned with `unique_zones` (the sorted distinct finite zone ids): per zone
    the most frequent valid value, smallest on ties, NaN for zones without valid cells (zonal.py:56-68
    `_stats_majority` = np.unique + argmax).

    int32 zones with float32-exact values take the (zone, value) pair-count kernel; anything else
    (non-integer or wide zone ids, float64 values that float32 cannot hold, more distinct pairs than
    the table may grow to) is grouped by one device sort."""
    import torch
    uz = np.asarray(unique_zones)
    out = np.full(len(uz), np.nan)
    if len(uz) == 0:
        return out
    vf = _float32_exact(values_t)
    if zones_t.dtype == torch.int32 and vf is not None:
        try:
            zone, val, c = pair_counts(zones_t, vf, nodata_values, comm, max_cap=_MAJORITY_PAIR_MAX_CAP)
            order = np.lexsort((val, -c, zone))      # per zone: highest count first, then smallest value
            zone, val = zone[order], val[order]
            first = np.r_[True, zone[1:] != zone[:-1]]
            pos = np.searchsorted(uz.astype(np.int64), zone[first])
            ok = (pos < len(uz)) & (uz.astype(np.int64)[np.minimum(pos, len(uz) - 1)] == zone[first])
            out[pos[ok]] = val[first][ok]
            return out
        except _PairTableOverflow:
            pass
    if comm is not None:
        raise NotImplementedError("'majority' over row stripes needs int32 zones and categorical float32-exact "
                                  "values (the sort-based path is single-GPU)")
    z = zones_t.reshape(-1)
    v = (vf if vf is not None else values_t.to(torch.float64)).reshape(-1) + 0.0   # -0.0 and 0.0 are one value
    ok = torch.isfinite(v)
    if nodata_values is not None:
        ok &= v != float(nodata_values)
    idx, hit = _zone_index(z, uz)
    ok &= hit
    return _majority_by_sort(idx[ok], v[ok], len(uz))


def _zone_index(z, sel):
    """(position in the sorted ids `sel`, cell's zone is in `sel`) for every cell of the flat zones `z`.
    Integer ids are matched as int64: float64 would merge ids above 2^53."""
    import torch
    if z.dtype.is_floating_point:
        ids_t = torch.as_tensor(np.asarray(sel, dtype=np.float64), device=z.device)
        zk = z.to(torch.float64)
    else:
        ids_t = torch.as_tensor(np.asarray(sel, dtype=np.int64), device=z.device)
        zk = z.to(torch.int64)
    idx = torch.searchsorted(ids_t, zk).clamp_(max=len(sel) - 1)
    return idx, ids_t[idx] == zk      # NaN zones match nothing


def _allreduce_partials(part, dev, comm):
    """Partials of the same zones on every rank combined over `comm`: SUM count / s1 / s2, MIN min, MAX max."""
    import torch
    import torch.distributed as dist
    t = {n: torch.as_tensor(a, device=dev) for n, a in part.items()}
    for n, op in (("count", dist.ReduceOp.SUM), ("s1", dist.ReduceOp.SUM), ("s2", dist.ReduceOp.SUM),
                  ("min", dist.ReduceOp.MIN), ("max", dist.ReduceOp.MAX)):
        dist.all_reduce(t[n], op=op, group=comm)
    return {n: v.cpu().numpy() for n, v in t.items()}


def allreduce_tables(ids, part, dev, comm):
    """Combine the per-stripe tables of all ranks: the id lists are all-gathered (a few KB), every
    rank scatters its partials into dense arrays over the sorted union of ids, and the dense
    arrays are combined with NCCL AllReduce (SUM for count / sums, MIN, MAX) -- SURVEY.md 8e."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(comm)
    n_local = torch.tensor([len(ids)], dtype=torch.int64, device=dev)
    counts = [torch.zeros(1, dtype=torch.int64, device=dev) for _ in range(world)]
    dist.all_gather(counts, n_local, group=comm)
    nmax = int(max(int(c.item()) for c in counts))
    pad = np.zeros(nmax, dtype=np.float64)
    pad[:len(ids)] = np.asarray(ids, dtype=np.float64)
    mine = torch.as_tensor(pad, device=dev)
    gathered = [torch.empty(nmax, dtype=torch.float64, device=dev) for _ in range(world)]
    dist.all_gather(gathered, mine, group=comm)
    union = np.unique(np.concatenate([g[:int(c.item())].cpu().numpy() for g, c in zip(gathered, counts)]))
    pos = np.searchsorted(union, np.asarray(ids, dtype=np.float64))
    dense = _empty_partials(len(union))
    for k in dense:
        dense[k][pos] = part[k]
    if len(union):
        dense = _allreduce_partials(dense, dev, comm)
    return union.astype(np.asarray(ids).dtype), dense


# Bound on the relative error of the kernel's float64 sums (count, s1, s2 are each a float64 sum over a
# zone's cells): 2^-40 = 8192 units in the last place, the worst case of a chain of 8192 roundings.
_SUM_REL_ERR = 2.0 ** -40


def one_pass_inaccurate(part, pivot):
    """True when the partials about the one global `pivot` may miss the accuracy of numpy's two-pass
    statistics (DESIGN 4.4).  With q = s2/n (mean square of v - pivot), the sums carry errors of about
    e*sqrt(q) in s1/n and 3*e*q in s2/n - (s1/n)^2 (e = _SUM_REL_ERR).  The one-pass result is kept when
    these stay ten times inside 1e-10 * (|mean| + M) for the mean and 1e-7 * var + 1e-12 * M^2 for the
    variance, M being the zone's largest |value|; otherwise the caller sums again about each zone's mean."""
    cnt = part["count"].astype(np.float64)
    ok = (cnt > 0) & (part["min"] != part["max"])      # constant zones: finalize is exact for them
    if not ok.any():
        return False
    n = cnt[ok]
    m1 = part["s1"][ok] / n
    q = part["s2"][ok] / n
    var = np.maximum(q - m1 * m1, 0.0)
    mean = pivot[ok] + m1 if np.ndim(pivot) else pivot + m1
    big = np.maximum(np.abs(part["min"][ok]), np.abs(part["max"][ok]))
    e = _SUM_REL_ERR
    with np.errstate(over="ignore", invalid="ignore"):
        bad_mean = e * np.sqrt(q) > 0.1 * 1e-10 * (np.abs(mean) + big)
        bad_var = 3.0 * e * q > 0.1 * (1e-7 * var + 1e-12 * big * big)
    return bool((bad_mean | bad_var).any())


def finalize(part, pivot, stats_funcs):
    """dict stat -> float64 column; zones without valid cells are NaN (zonal.py:153-162)."""
    cnt = part["count"].astype(np.float64)
    ok = cnt > 0
    const = part["min"] == part["max"]
    with np.errstate(invalid="ignore", divide="ignore"):
        m1 = part["s1"] / cnt
        cols = {}
        for s in stats_funcs:
            # a zone whose valid values are all equal (min == max) gets numpy's exact mean, sum and var
            if s == "mean":
                c = np.where(const, part["min"], pivot + m1)
            elif s == "sum":
                c = np.where(const, part["min"] * cnt, pivot * cnt + part["s1"])
            elif s in ("var", "std"):
                c = np.where(const, 0.0, np.maximum(part["s2"] / cnt - m1 * m1, 0.0))
                if s == "std":
                    c = np.sqrt(c)
            elif s == "count":
                c = cnt.copy()
            elif s == "max":
                c = part["max"].copy()
            elif s == "min":
                c = part["min"].copy()
            else:
                raise ValueError("Invalid stat name. %s option not supported." % s)
            c = np.where(ok, c, np.nan)
            cols[s] = c
    return cols


def _partial_columns(zt, vt, table, ids, part, pivot, names, nodata_values, comm, pos):
    """finalize(...) of `names` over the zones ids[pos] from hash_partials' results.
    mean / sum / std / var come from a second pass about each zone's own mean (numpy's two-pass statistics) for
    float64 rasters when std / var are asked for, and whenever the one-pass sums over these zones may be too
    inaccurate (zones far from the pivot for their spread)."""
    import torch
    sel_part = {n: a[pos] for n, a in part.items()}
    sel_pivot = np.full(len(sel_part["count"]), pivot)
    moments = [s for s in names if s in ("mean", "sum", "std", "var")]
    second = len(sel_pivot) > 0 and bool(moments) and \
        ((vt.dtype == torch.float64 and any(s in ("std", "var") for s in names)) or
         one_pass_inaccurate(sel_part, sel_pivot))
    cols = finalize(sel_part, sel_pivot, [s for s in names if not (second and s in moments)])
    if second:
        cnt = part["count"].astype(np.float64)
        with np.errstate(invalid="ignore", divide="ignore"):
            means = np.where(cnt > 0, pivot + part["s1"] / cnt, 0.0)
        part2 = second_pass_partials(zt, vt, table, ids, means, nodata_values, comm=comm)
        cols.update(finalize({n: a[pos] for n, a in part2.items()}, means[pos], moments))
    return cols


def _zone_columns(zt, vt, names, nodata_values, comm, zone_ids, keep_order=False):
    """(ids, cols): the zones `_select_zones(..., zone_ids, keep_order)` reports for the prepared zones `zt` and
    values `vt`, and one float64 column per built-in statistic of `names`, aligned with them."""
    table = {}
    present, part, pivot = hash_partials(zt, vt, nodata_values, comm=comm, table=table)
    ids, pos = _select_zones(present, zone_ids, keep_order)
    cols = _partial_columns(zt, vt, table, present, part, pivot, [s for s in names if s != "majority"],
                            nodata_values, comm, pos)
    if "majority" in names:
        cols["majority"] = majority_by_zone(zt, vt, present, nodata_values, comm=comm)[pos]
    return ids, cols


def _zone_table(ids, cols, names, zt, values, return_type):
    """A zone column and one column per name as a DataFrame, or, for any other `return_type`, every column
    broadcast back onto its zone's cells in the container of `values`."""
    if return_type == 'pandas.DataFrame':
        return pd.DataFrame({"zone": ids, **{s: cols[s] for s in names}})
    return like_container(_broadcast_back(cols, names, ids, zt), values)


def _stats_device(zones, values, zone_ids, stats_funcs, nodata_values, return_type='pandas.DataFrame',
                  comm=None):
    """Device runner (replaces zonal.py:335 `_stats_cupy`)."""
    zt = _prepare_zones(as_device_tensor(zones))
    vt = _prepare_values(as_device_tensor(values))
    if len(vt.shape) > 2:
        raise TypeError('3D inputs not supported for the device backend')
    names = list(stats_funcs)
    ids, cols = _zone_columns(zt, vt, names, nodata_values, comm, zone_ids)
    return _zone_table(ids, cols, names, zt, values, return_type)


def _broadcast_back(cols, names, sel, zt):
    """(len(names), H, W) float64 tensor: every statistic broadcast onto its zone's cells, NaN
    elsewhere (zonal.py:313-331)."""
    import torch
    out = torch.full((len(names), zt.numel()), float("nan"), dtype=torch.float64, device=zt.device)
    if len(sel):
        idx, hit = _zone_index(zt.reshape(-1), sel)
        for i, s in enumerate(names):
            table = torch.as_tensor(np.asarray(cols[s], dtype=np.float64), device=zt.device)
            out[i] = torch.where(hit, table[idx], out[i])
    return out.reshape(len(names), *zt.shape)


def _stats_custom(zones, values, zone_ids, stats_funcs, nodata_values, return_type='pandas.DataFrame',
                  host=False):
    """`stats_funcs` given as a dict of callables (zonal.py:640-642): the reference groups the cells
    by zone with an argsort and calls every function on the zone's valid values
    (`_calc_stats`, zonal.py:144-163).  Same here, with the grouping done by one stable device
    sort; the callables receive the zone's values in the raster's dtype -- numpy arrays for numpy
    rasters (`host`), device tensors otherwise -- and must return a scalar."""
    import torch
    zt = _prepare_zones(as_device_tensor(zones))
    vt = as_device_tensor(values).contiguous()
    if len(vt.shape) > 2:
        raise TypeError('3D inputs not supported for the device backend')
    for name, f in stats_funcs.items():
        if not callable(f):
            raise ValueError(name)
    z = zt.reshape(-1)
    v = vt.reshape(-1)
    zfinite = torch.isfinite(z) if z.dtype.is_floating_point else None
    sel, _ = _select_zones(torch.unique(z[zfinite] if zfinite is not None else z).cpu().numpy(), zone_ids)
    ok = torch.isfinite(v) if v.dtype.is_floating_point else torch.ones_like(v, dtype=torch.bool)
    if nodata_values is not None:
        ok &= v != nodata_values
    if zfinite is not None:
        ok &= zfinite
    zk, vk = z[ok], v[ok]
    order = torch.argsort(zk, stable=True)
    zs, vs = zk[order], vk[order]
    present, counts = torch.unique_consecutive(zs, return_counts=True)
    present, counts = present.cpu().numpy(), counts.cpu().numpy()
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]]) if len(counts) else np.zeros(0, np.int64)
    where = {zz: (int(a), int(a + c)) for zz, a, c in zip(present.tolist(), starts, counts)}
    groups = vs.cpu().numpy() if host else vs
    cols = {}
    for name, func in stats_funcs.items():
        col = np.full(len(sel), np.nan)
        for i, zz in enumerate(sel.tolist()):
            if zz in where:
                a, b = where[zz]
                col[i] = float(func(groups[a:b]))
        cols[name] = col
    return _zone_table(sel, cols, list(stats_funcs), zt, values, return_type)


def _stats_host(zones, values, zone_ids, stats_funcs, nodata_values, return_type='pandas.DataFrame'):
    """numpy runner (replaces zonal.py:280 `_stats_numpy`): upload, same device pass."""
    zt, vt = _device_tensor(zones), _device_tensor(values)
    if isinstance(stats_funcs, dict):
        res = _stats_custom(zt, vt, zone_ids, stats_funcs, nodata_values, return_type, host=True)
    else:
        res = _stats_device(zt, vt, zone_ids, stats_funcs, nodata_values, return_type)
    if return_type != 'pandas.DataFrame':
        return res.cpu().numpy()
    res["zone"] = res["zone"].astype(np.asarray(zones).dtype)
    return res


def stats(zones, values, zone_ids=None,
          stats_funcs=["mean", "max", "min", "sum", "std", "var", "count", "majority"],
          nodata_values=None, return_type='pandas.DataFrame', comm=None):
    """Per-zone summary statistics (zonal.py:422-667), same signature and defaults.

    `stats_funcs` as a list names built-in statistics: they come from one streaming pass over the
    raster (`majority` adds a second pass, so leave it out of the list when it is not needed).
    `stats_funcs` as a dict maps column names to callables, which are run per zone like the
    reference does (no built-in is ever substituted for a callable).  `comm` (optional
    torch.distributed group, not in the reference) marks `zones` and `values` as this rank's row
    stripe of a larger raster; custom callables are not available over stripes.
    """
    if isinstance(values, Dataset):
        if return_type != 'pandas.DataFrame':
            raise ValueError("return_type must be 'pandas.DataFrame' when values is a Dataset")
        dfs = []
        for var_name in values.data_vars:
            df = stats(zones, values[var_name], zone_ids, stats_funcs, nodata_values, 'pandas.DataFrame')
            df = df.rename(columns={c: f'{var_name}_{c}' for c in df.columns if c != 'zone'})
            dfs.append(df)
        result = dfs[0]
        for df in dfs[1:]:
            result = result.merge(df, on='zone', how='outer')
        return result

    validate_arrays(zones, values)
    for nm, arr in (("zones", zones), ("values", values)):
        dt = arr.data.dtype
        kind = getattr(dt, "kind", None)
        if kind is None:  # torch dtype
            ok = dt.is_floating_point or "int" in str(dt)
        else:
            ok = kind in "iuf"
        if not ok:
            raise ValueError("`%s` must be an array of integers or floats." % nm)

    if isinstance(stats_funcs, list):
        for s in stats_funcs:
            if s not in _DEFAULT_STATS:
                raise ValueError(f"Invalid stat name. {s} option not supported.")
        funcs = list(stats_funcs)
        names = funcs
    elif isinstance(stats_funcs, dict):
        funcs = dict(stats_funcs)
        names = list(funcs.keys())
        if comm is not None:
            raise NotImplementedError("custom statistics cannot be combined across row stripes; "
                                      "name built-in statistics in a list when `comm` is given")
    else:  # the reference falls through to an UnboundLocalError here; say what is wrong instead
        raise TypeError("`stats_funcs` must be a list of statistic names or a dict of callables")

    if comm is not None:
        result = _stats_device(zones.data, values.data, zone_ids, funcs, nodata_values, return_type, comm)
    else:
        device = _stats_custom if isinstance(funcs, dict) else _stats_device
        mapper = ArrayTypeFunctionMapping(
            numpy_func=lambda *a: _stats_host(*a, return_type=return_type),
            cupy_func=lambda *a: device(*a, return_type=return_type))
        result = mapper(values)(zones.data, values.data, zone_ids, funcs, nodata_values)

    if return_type == 'xarray.DataArray':
        coords = {'stats': names}
        coords.update(values.coords)
        return DataArray(result, coords=coords, dims=('stats',) + tuple(values.dims), attrs=values.attrs)
    return result


TOTAL_COUNT = '_total_count'


def _pivot_pairs(sel, cats, pz, pv, pc):
    """(zone, value, count) pairs -> per-zone totals (float32, like the reference) and a
    (len(cats), len(sel)) count matrix.  `cats` is sorted; zones outside `sel` are dropped.
    zonal.py:719-727: a selected category also collects the unselected categories between it and
    the previous selected one (the reference's `cat_start` only advances at selected categories);
    with all categories selected this is the plain per-category count."""
    total = np.zeros(len(sel), dtype=np.float32)
    counts = np.zeros((len(cats), len(sel)), dtype=np.int64)
    if len(sel) == 0 or len(pz) == 0:
        return total, counts
    sel_f = np.asarray(sel, dtype=np.float64)
    order = np.argsort(sel_f, kind="stable")
    pos = np.searchsorted(sel_f[order], pz.astype(np.float64), side="right") - 1   # last of equal ids
    pos[pos < 0] = 0
    hit = sel_f[order][pos] == pz
    row = order[pos]
    np.add.at(total, row[hit], pc[hit].astype(np.float32))      # unbuffered: pair order, like a loop
    if len(cats):
        bounds = np.asarray([float(c) for c in cats], dtype=np.float64)
        col = np.searchsorted(bounds, pv, side="left")
        keep = hit & (col < len(cats))
        np.add.at(counts, (col[keep], row[keep]), pc[keep])
    return total, counts


def _crosstab_3d(zones, values, zone_ids, cat_ids, layer, agg, nodata_values, comm):
    """3-D `values` (zonal.py:1096-1116, `_single_zone_crosstab_3d` :734-745): the categories are the
    coordinate values of dimension `layer`, and cell (zone, category) is statistic `agg` of that
    category's 2-D layer over the zone: the column is zonal.stats of that layer, zones in the order of `zone_ids`."""
    import torch
    if agg not in _DEFAULT_STATS:
        raise ValueError("`agg` method for 3D numpy backed data array must be one of following %s"
                         % (list(_DEFAULT_STATS),))
    if layer is None:
        layer = 0
    try:
        ldim = values.dims[layer]
        if ldim not in values.coords:
            raise KeyError(ldim)
        unique_cats = np.asarray(getattr(values.coords[ldim], "values", values.coords[ldim]))
    except (IndexError, KeyError, TypeError):
        raise ValueError("Invalid `layer`")
    axis = list(values.dims).index(ldim)
    vt = torch.movedim(_device_tensor(values.data), axis, 0)
    zt = _device_tensor(zones.data)
    if tuple(zt.shape) != tuple(vt.shape[1:]):
        raise ValueError("Incompatible shapes")
    zt = _prepare_zones(zt)
    if cat_ids is None:
        cats = list(unique_cats.tolist())
    else:
        cats = [c for c in cat_ids if c in unique_cats]
    cat_pos = {c: j for j, c in enumerate(unique_cats.tolist())}
    d = {}
    for c in cats:
        ids, cols = _zone_columns(zt, _prepare_values(vt[cat_pos[c]]), [agg], nodata_values, comm, zone_ids,
                                  keep_order=True)
        col = cols[agg]
        if agg == "count":          # np.ma.count of an empty selection is 0, and the column is integer
            col = np.where(np.isnan(col), 0, col).astype(np.int64)
        d[c] = col
    if not cats:                    # the zones alone: every zone is met, even by a pass without valid values
        ids, _ = _zone_columns(zt, torch.full(zt.shape, float("nan"), device=zt.device), [], None, comm, zone_ids,
                               keep_order=True)
    return pd.DataFrame({"zone": ids, **d})


def crosstab(zones, values, zone_ids=None, cat_ids=None, layer=None, agg="count", nodata_values=None, comm=None):
    """Cross-tabulation of a `values` raster by zone (zonal.py:922-1155): a `zone` column and one column
    per category.  2-D values: cell counts (or percentages) of the categorical values per zone, built on
    the (zone, value) pair histogram of xrs_zonal_pair_count.  3-D values: statistic `agg` of every
    category layer per zone (`layer` names the category dimension)."""
    if not isinstance(zones, DataArray):
        raise TypeError("zones must be instance of DataArray")
    if not isinstance(values, DataArray):
        raise TypeError("values must be instance of DataArray")
    if zones.ndim != 2:
        raise ValueError("zones must be 2D")
    if values.ndim not in (2, 3):
        raise ValueError("`values` must use either 2D or 3D coordinates.")
    if values.ndim == 3:
        return _crosstab_3d(zones, values, zone_ids, cat_ids, layer, agg, nodata_values, comm)
    validate_arrays(zones, values)
    if agg not in ("percentage", "count"):
        raise ValueError("`agg` method for 2D data array must be one of following ['percentage', 'count']")
    zt, vt = _prepare_zones(_device_tensor(zones.data)), _device_tensor(values.data)
    vt_f = _prepare_values(vt)
    present, _, _ = hash_partials(zt, vt_f, None, comm=comm)
    zi, vf = _pair_inputs(zt, vt_f)
    try:
        pz, pv, pc = pair_counts(zi, vf, nodata_values, comm=comm)
    except _PairTableOverflow:
        raise NotImplementedError("crosstab: more than 64M distinct (zone, category) pairs")
    vdtype = np.dtype(str(vt.dtype).replace("torch.", "")) if not isinstance(values.data, np.ndarray) else values.data.dtype
    unique_cats = np.unique(pv).astype(vdtype)
    if cat_ids is None:
        cats = unique_cats
    else:
        cats = [c for c in cat_ids if c in unique_cats]
    sel, _ = _select_zones(present, zone_ids, keep_order=True)
    cats = sorted(cats)
    total, counts = _pivot_pairs(sel, cats, pz, pv, pc)
    table = {c: counts[j] for j, c in enumerate(cats)}
    d = {"zone": sel}
    if agg == "percentage":
        total[total == 0] = np.nan
        for c in cats:
            d[c] = table[c] / total * 100
    else:
        for c in cats:
            d[c] = table[c]
    return pd.DataFrame(d)


# ----------------------------------------------------------------------------- regions, trim, crop
def regions(raster, neighborhood=4, name="regions"):
    """Number the connected regions of cells with close values (zonal.py:1552-1640 of the reference).

    Cells join their 4 or 8 neighbours when |neighbour - cell| <= 1e-08 + 1e-05 |cell|, evaluated as the
    reference's numba kernel evaluates it for the cell type.  Every cell gets the label the reference's two-pass
    scan gives it, in the raster's cell type (labels are not renumbered, so they may have gaps); NaN cells stay
    NaN, and a bool raster gives all True.  Labels are exact in int64 before the one cast to the cell type, where
    the reference's own labels wrap or round once they pass the type's range (DESIGN.md section 4.12)."""
    import torch
    if neighborhood not in (4, 8):
        raise ValueError("`neighborhood` value must be either 4 or 8)")
    data = raster.data
    t, code = device_cells(data, "regions", "as-is")
    H, W = t.shape
    out = torch.empty((H, W), dtype=t.dtype, device=t.device)
    if H and W:
        scratch, size = device_scratch("xrs_zonal_regions_scratch_bytes", H, W, device=t.device, what="regions")
        call_on(t, "xrs_zonal_regions", ptr(t), code, pitch(t), H, W, neighborhood, ptr(out), pitch(out),
                ptr(scratch), size)
    return DataArray(to_container(out, data), name=name, dims=raster.dims, coords=raster.coords, attrs=raster.attrs)


def _bounds(data, values, mode, what):
    """(top, bottom, left, right) as the reference's _trim (mode 0) or _crop (mode 1) finds them: the first and
    last rows and columns holding a cell that equals none of `values` (trim) or one of them (crop), and
    (rows - 1, 0, cols - 1, 0) when no cell does."""
    import torch
    t, code = device_cells(data, what, "as-is")
    H, W = t.shape
    vals = list(values)
    # numba types a list of ints as int64 and compares integer cells with them exactly; any float makes it float64
    ints = all(isinstance(v, (int, np.integer, np.bool_)) for v in vals)
    dv = torch.tensor([float(v) for v in vals], dtype=torch.float64, device=t.device)
    iv = torch.tensor([int(v) for v in vals], dtype=torch.int64, device=t.device) if ints and vals else None
    out4 = torch.empty(4, dtype=torch.int64, device=t.device)
    call_on(t, "xrs_zonal_bounds", ptr(t), code, pitch(t), H, W, mode, ptr(dv) if vals else None,
            ptr(iv) if iv is not None else None, len(vals), ptr(out4))
    top, bottom, left, right = out4.cpu().tolist()
    if bottom < 0:
        return max(H - 1, 0), 0, max(W - 1, 0), 0
    return top, bottom, left, right


def _window(raster, top, bottom, left, right, name):
    """raster[top:bottom + 1, left:right + 1] with its coordinates sliced alike (the shim DataArray has no
    positional indexing)."""
    rs, cs = slice(top, bottom + 1), slice(left, right + 1)
    by_dim = dict(zip(raster.dims, (rs, cs)))
    coords = {}
    for k, v in raster.coords.items():
        dims = getattr(v, "dims", None)
        v = v.data if dims is not None else v
        shape = tuple(getattr(v, "shape", ()))
        if dims is None:   # shim coordinates are bare arrays: a 1-D one named after a dimension runs along it
            dims = (k,) if len(shape) == 1 and k in by_dim else tuple(raster.dims) if shape == raster.shape else ()
        if len(dims) == len(shape) and any(d in by_dim for d in dims):
            v = DataArray(v[tuple(by_dim.get(d, slice(None)) for d in dims)], dims=dims)
        coords[k] = v
    return DataArray(raster.data[rs, cs], name=name, dims=raster.dims, coords=coords, attrs=raster.attrs)


def trim(raster, values=(np.nan,), name="trim"):
    """Drop the edge rows and columns that hold only `values` (zonal.py:1734-1842 of the reference).

    Cells equal a value as in the reference's numba loop: integer cells and integer values exactly, anything
    with a float in float64, NaN never (so the default trims nothing).  When every cell is one of the values the
    reference's bounds (rows - 1, 0, cols - 1, 0) give an empty result unless that side has length 1."""
    top, bottom, left, right = _bounds(raster.data, values, 0, "trim")
    return _window(raster, top, bottom, left, right, name)


def crop(zones, values, zones_ids, name="crop"):
    """Cut `values` to the rows and columns between the first and last cells of `zones` equal to one of
    `zones_ids` (zonal.py:1943-2062 of the reference); equality as in trim."""
    top, bottom, left, right = _bounds(zones.data, zones_ids, 1, "crop")
    return _window(values, top, bottom, left, right, name)


# ----------------------------------------------------------------------------- canvas size
_FULL_EXTENTS = {"Mercator": ((-20e6, 20e6), (-20e6, 20e6)), "Geographic": ((-180, 180), (-90, 90))}


def get_full_extent(crs):
    """((min_x, max_x), (min_y, max_y)) of the 'Mercator' or 'Geographic' projection; KeyError for others."""
    return _FULL_EXTENTS[crs]


def suggest_zonal_canvas(smallest_area, x_range, y_range, crs="Mercator", min_pixels=25):
    """(height, width) of a canvas over x_range x y_range on which a polygon of `smallest_area` covers about
    `min_pixels` pixels, with the pixels as square as the projection's full extent allows (zonal.py:1304-1403
    of the reference, in its float operations)."""
    (x0, x1), (y0, y1) = get_full_extent(crs)
    aspect = (x1 - x0) / (y1 - y0)
    pixels = (x1 - x0) * (y1 - y0) / (smallest_area / min_pixels)
    h = math.sqrt(pixels / aspect)
    w = aspect * h
    return int(h * (y_range[1] - y_range[0]) / (y1 - y0)), int(w * (x_range[1] - x_range[0]) / (x1 - x0))

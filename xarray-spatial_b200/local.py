"""xrspatial.local on the CUDA backend (reference: local.py): cell-by-cell functions over a Dataset's variables.

Every function reads its K variables cell by cell in one kernel (csrc/local.cu) whose per-cell rule
(csrc/local_rule.cuh) restates what the reference computes on the cell's K Python scalars, value for value; combine
numbers the distinct tuples through a device hash table.  A Dataset of numpy variables is uploaded and gives a
numpy-backed DataArray; a Dataset of CUDA tensors gives a tensor-backed one.  DESIGN.md section 4.13 lists the
semantics and the deviations.
"""
import ctypes

import numpy as np

from . import _lib
from ._xr import DataArray, Dataset
from .utils import call_on, device_2d, device_scratch, pitch, ptr, raster_cells, uint64_as_int64

try:
    import torch
except ImportError:  # pragma: no cover
    torch = None

# the reference's statistic names, in its order (its error message lists them), and the rule's op codes
funcs = {'max': 4, 'mean': 1, 'median': 2, 'min': 3, 'std': 5, 'sum': 0}
OPS = dict(lesser_frequency=6, equal_frequency=7, greater_frequency=8, lowest_position=9, highest_position=10,
           popularity=11, rank=12)
FLOAT, INT, BOOL = 0, 1, 2                               # the stack's array kind (np.array(tuple).dtype)
FLAG_NAN, FLAG_INDEX, FLAG_TYPE, FLAG_FLOAT, FLAG_INT = 1, 2, 4, 8, 16
_COUNTS = {6, 7, 8, 9, 10}                               # counts and positions: int64, or float64 with NaN


_NOT_DATASET = "Expected raster to be a 'xarray.Dataset'. Received '%s' instead."
_BAD_FUNC = "%s is not supported. The supported types are '%s'."
_REF_NOT_STR = "Expected ref_var to be a 'str'. Received '%s' instead."
_VARS_MISSING = "raster must contain all the variables of data_vars. The variables available are '%s'."


def _check(raster, data_vars, ref_var=None, has_ref=False, func=None):
    """The selected variable names, after the argument checks local.py makes, with its exception types and messages
    and in its order: the raster, func, ref_var, then data_vars."""
    if not isinstance(raster, Dataset):
        raise TypeError(_NOT_DATASET % type(raster).__name__)
    if func is not None and func not in funcs:
        raise ValueError(_BAD_FUNC % (func, list(funcs)))
    names = list(raster.data_vars)
    if has_ref and not isinstance(ref_var, str):
        raise TypeError(_REF_NOT_STR % type(ref_var).__name__)
    if has_ref and ref_var not in names:
        raise ValueError("raster must contain ref_var.")
    if not data_vars:   # None or empty: every variable but the ref
        selected = [n for n in names if not (has_ref and n == ref_var)]
    elif not isinstance(data_vars, list) or any(not isinstance(v, str) for v in data_vars):
        raise TypeError("Expected data_vars to be a list of string.")
    elif any(v not in names for v in data_vars):
        raise ValueError(_VARS_MISSING % names)
    elif has_ref and ref_var in data_vars:
        raise ValueError("ref_var must not be an element of data_vars.")
    else:
        selected = data_vars
    if len(selected) == 1:
        # np.nditer over one array yields 0-d arrays, which the reference then iterates
        raise TypeError("iteration over a 0-d array")
    return selected


def _cells(data, name):
    """(cells as the kernel reads them, their xrs_dtype code, True for float16 cells carried as float32)."""
    what = "local: variable %r" % name
    dt = str(getattr(data, "dtype", "")).replace("torch.", "")
    if dt == "float16":   # exact in float32; a float16 ref still compares in float16
        data = data.astype(np.float32) if isinstance(data, np.ndarray) else data.float()
        cells, code = raster_cells(data, what, "as-is")
        return cells, code, True
    cells, code = raster_cells(data, what, "as-is")
    if dt == "uint64":
        cells = uint64_as_int64(cells, what)   # still read as uint64 cells (code), below 2**63
    return cells, code, False


class _Stack:
    """The selected variables (and ref) checked, with their codes, on the device (or, for the host build of the
    rule, as CPU tensors)."""

    def __init__(self, raster, data_vars, ref_var=None, device=True):
        arrays = [raster[v].data for v in data_vars] + ([raster[ref_var].data] if ref_var is not None else [])
        self.host = all(isinstance(a, np.ndarray) for a in arrays)
        prepared = [_cells(a, n) for a, n in zip(arrays, list(data_vars) + [ref_var])]
        shapes = {tuple(c.shape) for c, _, _ in prepared}
        if len(shapes) != 1:
            raise ValueError("local: every variable must have the same 2-D shape, got %s" % sorted(shapes))
        self.H, self.W = shapes.pop()
        self.tensors = [device_2d(c) if device else torch.from_numpy(np.ascontiguousarray(c)) for c, _, _ in prepared]
        self.codes = [code for _, code, _ in prepared]
        self.f16 = [f for _, _, f in prepared]
        self.K = len(data_vars)
        kinds = {BOOL if c == _lib.ZONAL_CELLS["bool"] else
                 FLOAT if c in (_lib.ZONAL_CELLS["float32"], _lib.ZONAL_CELLS["float64"]) else INT
                 for c in self.codes[:self.K]}
        self.ak = FLOAT if FLOAT in kinds else (INT if INT in kinds else BOOL)
        devices = {t.device for t in self.tensors}
        if len(devices) > 1:
            raise ValueError("local: every variable must be on one device, got %s" % sorted(map(str, devices)))
        self.device = self.tensors[0].device

    def descriptors(self, tensors):
        """K layers as the host array {pointer, pitch, dtype} per layer the entry points take, and a device
        buffer for their copy."""
        rows = [(t.data_ptr(), pitch(t), c) for t, c in zip(tensors, self.codes)]
        host = (ctypes.c_int64 * (3 * len(rows)))(*[v for r in rows for v in r])
        return host, torch.empty(3 * len(rows), dtype=torch.int64, device=self.device)

    def container(self, out):
        return out.cpu().numpy() if self.host else out


def _finish(op, ak, bits, kinds, flags, ref_type=None):
    """The result array the reference builds from the per-cell results: `bits` int64 (H, W), `kinds` the per-cell
    kinds (rank and popularity), `flags` the OR of the cells' flags."""
    if flags & FLAG_TYPE:
        raise TypeError("list indices must be integers or slices, not numpy.%s" % ref_type)
    if flags & FLAG_INDEX:
        raise IndexError("list index out of range")
    as_float = bits.view(torch.float64)
    if op in (1, 2, 5) or (op in (0, 3, 4) and ak == FLOAT):
        return as_float
    if op in (0, 3, 4):
        return bits != 0 if (ak == BOOL and op != 0) else bits
    if op in _COUNTS or op == "combine":
        if flags & FLAG_NAN:
            return torch.where(bits < 0, torch.full_like(as_float, float("nan")), bits.to(torch.float64))
        return bits
    if flags & (FLAG_NAN | FLAG_FLOAT):
        return torch.where(kinds == FLOAT, as_float, bits.to(torch.float64))
    return bits if flags & FLAG_INT else bits != 0


def _ref_type(stack):
    if stack.f16[-1]:
        return "float16"
    return {_lib.ZONAL_CELLS["float32"]: "float32", _lib.ZONAL_CELLS["float64"]: "float64"}.get(stack.codes[-1])


def _run(op, raster, data_vars, ref_var=None):
    s = _Stack(raster, data_vars, ref_var)
    H, W = s.H, s.W
    bits = torch.empty((H, W), dtype=torch.int64, device=s.device)
    kinds = torch.empty((H, W), dtype=torch.uint8, device=s.device) if op in (11, 12) else None
    flags = torch.zeros(1, dtype=torch.int32, device=s.device)
    if H and W:
        host, dev = s.descriptors(s.tensors[:s.K])
        ref = s.tensors[s.K] if ref_var is not None else None
        call_on(bits, "xrs_local_cells", host, s.K, ptr(dev), H, W, op, s.ak, None if ref is None else ptr(ref),
                0 if ref is None else pitch(ref), 0 if ref is None else s.codes[s.K],
                int(ref is not None and s.f16[s.K]), ptr(bits), pitch(bits), None if kinds is None else ptr(kinds), W,
                ptr(flags))
    out = _finish(op, s.ak, bits, kinds, int(flags.item()), _ref_type(s) if ref_var is not None else None)
    return DataArray(s.container(out))


def _gather(t, code, rows, cols):
    """t[rows, cols] as Python scalars; uint16 and uint32 cells are gathered through their signed view."""
    for name, signed, mask in (("uint16", torch.int16, 0xFFFF), ("uint32", torch.int32, 0xFFFFFFFF)):
        if code == _lib.ZONAL_CELLS[name]:
            return (t.view(signed)[rows, cols].to(torch.int64) & mask).tolist()
    return t[rows, cols].tolist()


def _combine(raster, data_vars):
    s = _Stack(raster, data_vars)
    H, W = s.H, s.W
    ids = torch.empty((H, W), dtype=torch.int64, device=s.device)
    flags = torch.zeros(1, dtype=torch.int32, device=s.device)
    key = {}
    if H and W:
        host, dev = s.descriptors(s.tensors)
        scratch, nbytes = device_scratch("xrs_local_combine_scratch_bytes", H, W, device=s.device, what="combine")
        table = scratch[:nbytes].view(torch.int64)
        args = [host, s.K, ptr(dev), H, W]
        call_on(ids, "xrs_local_combine", *args, 0, ptr(scratch), nbytes, None, ptr(ids), pitch(ids), ptr(flags))
        # the occupied slots hold each tuple's first cell: number them in that order
        slots = torch.nonzero(table != torch.iinfo(torch.int64).max).flatten()
        reps, order = torch.sort(table[slots])
        table[slots[order]] = -1 - torch.arange(len(reps), device=s.device)
        call_on(ids, "xrs_local_combine", *args, 1, ptr(scratch), nbytes, ptr(reps), ptr(ids), pitch(ids), ptr(flags))
        rows, cols = reps // W, reps % W
        columns = [_gather(t, code, rows, cols) for t, code in zip(s.tensors, s.codes)]
        key = {i + 1: tup for i, tup in enumerate(zip(*columns))}
    out = _finish("combine", s.ak, ids, None, int(flags.item()))
    return DataArray(s.container(out), attrs=dict(key=key))


def cell_stats(raster, data_vars=None, func='sum'):
    """Statistic `func` (max, mean, median, min, std or sum) of the variables, cell by cell (local.py:16-79)."""
    data_vars = _check(raster, data_vars, func=func)
    return _run(funcs[func], raster, data_vars)


def combine(raster, data_vars=None):
    """A number for each distinct combination of the variables' values, 1, 2, ... in order of first occurrence;
    attrs['key'] maps each number to its combination (local.py:82-164)."""
    data_vars = _check(raster, data_vars)
    return _combine(raster, data_vars)


def lesser_frequency(raster, ref_var, data_vars=None):
    """How many variables are below ref_var, cell by cell (local.py:167-247)."""
    data_vars = _check(raster, data_vars, ref_var, True)
    return _run(OPS["lesser_frequency"], raster, data_vars, ref_var)


def equal_frequency(raster, ref_var, data_vars=None):
    """How many variables equal ref_var, cell by cell (local.py:250-330)."""
    data_vars = _check(raster, data_vars, ref_var, True)
    return _run(OPS["equal_frequency"], raster, data_vars, ref_var)


def greater_frequency(raster, ref_var, data_vars=None):
    """How many variables are above ref_var, cell by cell (local.py:333-413)."""
    data_vars = _check(raster, data_vars, ref_var, True)
    return _run(OPS["greater_frequency"], raster, data_vars, ref_var)


def lowest_position(raster, data_vars=None):
    """1-based index of the first variable holding the cell's least value (local.py:416-478)."""
    data_vars = _check(raster, data_vars)
    return _run(OPS["lowest_position"], raster, data_vars)


def highest_position(raster, data_vars=None):
    """1-based index of the first variable holding the cell's largest value (local.py:481-543)."""
    data_vars = _check(raster, data_vars)
    return _run(OPS["highest_position"], raster, data_vars)


def popularity(raster, ref_var, data_vars=None):
    """The ref_var-th smallest distinct value of the cell, where some value repeats (local.py:546-633)."""
    data_vars = _check(raster, data_vars, ref_var, True)
    return _run(OPS["popularity"], raster, data_vars, ref_var)


def rank(raster, ref_var, data_vars=None):
    """The ref_var-th smallest value of the cell (local.py:636-716)."""
    data_vars = _check(raster, data_vars, ref_var, True)
    return _run(OPS["rank"], raster, data_vars, ref_var)

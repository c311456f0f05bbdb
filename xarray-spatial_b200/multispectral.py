"""xrspatial.multispectral band indices on the CUDA backend (reference: multispectral.py).

ndvi / savi / evi (named by the north star) plus arvi, gci, sipi, ebbi, nbr, nbr2, ndmi, which
share the same per-cell pattern.  Inputs are cast to float32 like the reference
(`.astype('f4')`, e.g. multispectral.py:727); outputs are float32 with NaN where the
denominator is zero.  `true_color` is out of scope (SURVEY.md section 2 row 8).
"""
import ctypes

import numpy as np

from ._xr import DataArray
from .dataset_support import supports_dataset_bands
from .utils import ArrayTypeFunctionMapping, as_device_tensor, call_on, like_container, ptr, validate_arrays


def _band_device(fn_name, bands, scalars=()):
    """Elementwise device call: bands are device arrays of equal shape."""
    import torch
    ts = []
    for b in bands:
        t = as_device_tensor(b)
        if t.dtype != torch.float32:
            t = t.to(torch.float32)
        ts.append(t.contiguous())
    out = torch.empty(ts[0].shape, dtype=torch.float32, device=ts[0].device)
    n = out.numel()
    if n:
        call_on(out, fn_name, *map(ptr, ts), *[s if isinstance(s, ctypes.c_int) else float(s) for s in scalars],
                ptr(out), n)
    return like_container(out, bands[0])


def _band_host(fn_name, bands, scalars=()):
    """numpy bands: upload, run the device kernel, download (torch is only the copy engine)."""
    import torch
    from . import _hostmem
    dev = [torch.from_numpy(np.ascontiguousarray(b, dtype=np.float32)).cuda(non_blocking=True) for b in bands]
    res = _band_device(fn_name, dev, scalars)
    out = _hostmem.empty(tuple(res.shape), np.float32)
    torch.from_numpy(out).copy_(res)
    return out


def _mapper(fn_name):
    return ArrayTypeFunctionMapping(
        numpy_func=lambda *a: _band_host(fn_name, a[:_NB[fn_name]], a[_NB[fn_name]:]),
        cupy_func=lambda *a: _band_device(fn_name, a[:_NB[fn_name]], a[_NB[fn_name]:]))


_NB = {"xrs_normalized_ratio_f32": 2, "xrs_savi_f32": 2, "xrs_evi_f32": 3, "xrs_arvi_f32": 3,
       "xrs_gci_f32": 2, "xrs_sipi_f32": 3, "xrs_ebbi_f32": 3}


# Soil-factor types for which the reference's Numba kernel sums `nir + red + soil_factor` in float32; every
# other accepted type (Python float and int, np.float64, np.int32, np.int64 and the unsigned types from uint16
# up) gives a float64 sum.  NumPy's promotion rules do not give this table (float32 + uint16 is float32 in
# NumPy, float64 in Numba), so it is pinned type by type by tests/golden/multispectral_edges.npz.
_SAVI_F32_SUM = (np.float32, np.int8, np.int16, np.uint8, np.bool_, bool)


def _wrap(out, like, name):
    return DataArray(out, name=name, coords=like.coords, dims=like.dims, attrs=like.attrs)


def _normalized_ratio(a_agg, b_agg, name):
    validate_arrays(a_agg, b_agg)
    out = _mapper("xrs_normalized_ratio_f32")(a_agg)(a_agg.data, b_agg.data)
    return _wrap(out, a_agg, name)


@supports_dataset_bands(nir='nir_agg', red='red_agg')
def ndvi(nir_agg, red_agg, name='ndvi'):
    """(nir - red) / (nir + red)  (multispectral.py:653-733)."""
    return _normalized_ratio(nir_agg, red_agg, name)


@supports_dataset_bands(nir='nir_agg', swir2='swir2_agg')
def nbr(nir_agg, swir2_agg, name='nbr'):
    """(nir - swir2) / (nir + swir2)  (multispectral.py:476-558)."""
    return _normalized_ratio(nir_agg, swir2_agg, name)


@supports_dataset_bands(swir1='swir1_agg', swir2='swir2_agg')
def nbr2(swir1_agg, swir2_agg, name='nbr2'):
    """(swir1 - swir2) / (swir1 + swir2)  (multispectral.py:561-649)."""
    return _normalized_ratio(swir1_agg, swir2_agg, name)


@supports_dataset_bands(nir='nir_agg', swir1='swir1_agg')
def ndmi(nir_agg, swir1_agg, name='ndmi'):
    """(nir - swir1) / (nir + swir1)  (multispectral.py:737-822)."""
    return _normalized_ratio(nir_agg, swir1_agg, name)


@supports_dataset_bands(nir='nir_agg', red='red_agg')
def savi(nir_agg, red_agg, soil_factor=1.0, name='savi'):
    """(nir - red) / ((nir + red + L) * (1 + L)), L in [-1, 1]  (multispectral.py:927-1009)."""
    validate_arrays(red_agg, nir_agg)
    if not -1.0 <= soil_factor <= 1.0:
        raise ValueError("soil factor must be between [-1.0, 1.0]")
    f32_sum = ctypes.c_int(int(isinstance(soil_factor, _SAVI_F32_SUM)))
    out = _mapper("xrs_savi_f32")(red_agg)(nir_agg.data, red_agg.data, soil_factor, f32_sum)
    return _wrap(out, nir_agg, name)


@supports_dataset_bands(nir='nir_agg', red='red_agg', blue='blue_agg')
def evi(nir_agg, red_agg, blue_agg, c1=6.0, c2=7.5, soil_factor=1.0, gain=2.5, name='evi'):
    """G * (nir - red) / (nir + c1*red - c2*blue + L)  (multispectral.py:226-342)."""
    if not red_agg.shape == nir_agg.shape == blue_agg.shape:
        raise ValueError("input layers expected to have equal shapes")
    if not isinstance(c1, (float, int)):
        raise ValueError("c1 must be numeric")
    if not isinstance(c2, (float, int)):
        raise ValueError("c2 must be numeric")
    if soil_factor > 1.0 or soil_factor < -1.0:
        raise ValueError("soil factor must be between [-1.0, 1.0]")
    if gain < 0:
        raise ValueError("gain must be greater than 0")
    validate_arrays(nir_agg, red_agg, blue_agg)
    out = _mapper("xrs_evi_f32")(red_agg)(nir_agg.data, red_agg.data, blue_agg.data, c1, c2, soil_factor, gain)
    return _wrap(out, nir_agg, name)


@supports_dataset_bands(nir='nir_agg', red='red_agg', blue='blue_agg')
def arvi(nir_agg, red_agg, blue_agg, name='arvi'):
    """(nir - 2*red + blue) / (nir + 2*red + blue)  (multispectral.py:79-172)."""
    validate_arrays(red_agg, nir_agg, blue_agg)
    out = _mapper("xrs_arvi_f32")(red_agg)(nir_agg.data, red_agg.data, blue_agg.data)
    return _wrap(out, nir_agg, name)


@supports_dataset_bands(nir='nir_agg', green='green_agg')
def gci(nir_agg, green_agg, name='gci'):
    """nir / green - 1  (multispectral.py:392-472)."""
    validate_arrays(nir_agg, green_agg)
    out = _mapper("xrs_gci_f32")(nir_agg)(nir_agg.data, green_agg.data)
    return _wrap(out, nir_agg, name)


@supports_dataset_bands(nir='nir_agg', red='red_agg', blue='blue_agg')
def sipi(nir_agg, red_agg, blue_agg, name='sipi'):
    """(nir - blue) / (nir - red)  (multispectral.py:1066-1157)."""
    validate_arrays(red_agg, nir_agg, blue_agg)
    out = _mapper("xrs_sipi_f32")(red_agg)(nir_agg.data, red_agg.data, blue_agg.data)
    return _wrap(out, nir_agg, name)


@supports_dataset_bands(red='red_agg', swir='swir_agg', tir='tir_agg')
def ebbi(red_agg, swir_agg, tir_agg, name='ebbi'):
    """(swir - red) / (10 * sqrt(swir + tir))  (multispectral.py:1209-1333)."""
    validate_arrays(red_agg, swir_agg, tir_agg)
    out = _mapper("xrs_ebbi_f32")(red_agg)(red_agg.data, swir_agg.data, tir_agg.data)
    return _wrap(out, red_agg, name)

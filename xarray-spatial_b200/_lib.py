"""ctypes binding of libxrs_b200.so (include/xrs_b200.h).

There is no CPU fallback: if the shared library is missing or no CUDA device is usable the
product raises (RuntimeError) instead of computing on the host.
"""
import ctypes
import os

HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(HERE, "libxrs_b200.so")

XRS_OK, XRS_EINVAL, XRS_ECUDA, XRS_EUNSUPPORTED, XRS_ENOMEM = 0, -1, -2, -3, -4
OPS = dict(slope=0, aspect=1, curvature=2, hillshade=3, focal_mean=4, convolve=5, focal_stat=6)
STATS = dict(mean=0, sum=1, min=2, max=3, std=4, range=5, var=6)
DTYPES = dict(float32=0, float64=1, int32=2, int64=3, int16=4, uint16=5)
# every cell type xrs_zonal_regions and xrs_zonal_bounds read as they are
ZONAL_CELLS = dict(DTYPES, int8=6, uint8=7, uint32=8, uint64=9, bool=10)

_lib = None

c_i64 = ctypes.c_int64
c_dbl = ctypes.c_double
c_int = ctypes.c_int
c_vp = ctypes.c_void_p


class XrsError(RuntimeError):
    pass


def _declare(lib):
    P, I64, D, I = c_vp, c_i64, c_dbl, c_int
    sig = {
        "xrs_abi_version": [],
        "xrs_device_count": [ctypes.POINTER(I)],
        "xrs_device_sm_count": [I, ctypes.POINTER(I)],
        "xrs_slope_f32": [P, I64, P, I64, I64, I64, D, D, P],
        "xrs_aspect_f32": [P, I64, P, I64, I64, I64, P],
        "xrs_curvature_f32": [P, I64, P, I64, I64, I64, D, P],
        "xrs_hillshade_f32": [P, I64, P, I64, I64, I64, D, D, P],
        "xrs_surface_suite_f32": [P, I64, P, P, P, P, I64, I64, I64, D, D, D, D, P],
        "xrs_geodesic": [P, I, I64, P, P, I, P, I64, I64, I64, D, I, P],
        "xrs_surface_typed": [I, P, I, I64, P, I64, I64, I64, P, P],
        "xrs_focal_mean_f32": [P, I64, P, I64, I64, I64, P, I, P],
        "xrs_focal_mean_f64": [P, I64, P, I64, I64, I64, P, I, P],
        "xrs_focal_mean_f32_f64": [P, I64, P, I64, I64, I64, P, I, P],
        "xrs_convolve2d_f32": [P, I64, P, I64, I64, I64, P, I, I, P],
        "xrs_focal_stat_f32": [P, I64, P, I64, I64, I64, P, I, I, I, P],
        "xrs_focal_stats_multi_f32": [P, I64, P, I64, I64, I64, I64, P, I, I, P, I, P],
        "xrs_global_stats_f32": [P, I64, D, P, P],
        "xrs_hotspots_classify_f32": [P, I64, D, D, P, P],
        "xrs_normalized_ratio_f32": [P, P, P, I64, P],
        "xrs_savi_f32": [P, P, D, I, P, I64, P],
        "xrs_evi_f32": [P, P, P, D, D, D, D, P, I64, P],
        "xrs_arvi_f32": [P, P, P, P, I64, P],
        "xrs_gci_f32": [P, P, P, I64, P],
        "xrs_sipi_f32": [P, P, P, P, I64, P],
        "xrs_ebbi_f32": [P, P, P, P, I64, P],
        "xrs_zonal_hash_run": [P, I, P, I, I64, I64, I, D, I, D, P, P, P, P, P, P, I, P, I, P, P],
        "xrs_zonal_hash_second_pass": [P, I, P, I, I64, I64, I, D, P, P, P, P, P, P, P, I, P, I, P, P],
        "xrs_zonal_pair_count": [P, P, I64, I64, I, D, P, P, I, P, P],
        "xrs_proximity_scratch_bytes": [I64, I64, I, ctypes.POINTER(I64)],
        "xrs_proximity": [P, I, I64, I64, I64, P, P, P, I, D, I, I, P, I64, P, I64, I, P],
        "xrs_viewshed_scratch_bytes": [I64, I64, ctypes.POINTER(I64)],
        "xrs_viewshed": [P, I, I64, I64, I64, I64, I64, D, D, D, D, P, I64, P, I64, P],
        "xrs_a_star_scratch_bytes": [I64, I64, ctypes.POINTER(I64)],
        "xrs_a_star_search": [P, I, I64, I64, I64, P, I, I, I64, I64, I64, I64, P, I64, P, I64,
                              ctypes.POINTER(I64), P],
        "xrs_a_star_snap": [P, I, I64, I64, I64, P, I, I64, I64, ctypes.POINTER(I64), ctypes.POINTER(I64), P, I64, P],
        "xrs_perm_tables_scratch_bytes": [I, I64, ctypes.POINTER(I64)],
        "xrs_perm_tables": [P, I, I64, P, P, I64, ctypes.POINTER(I64), P],
        "xrs_noise_scratch_bytes": [I64, I64, I, ctypes.POINTER(I64)],
        "xrs_noise": [P, I, I64, I64, I64, P, P, P, I, D, P, I64, P, P, I64, P],
        "xrs_classify_cells": [P, I, I64, I64, I64, I, P, P, I, P, I64, P],
        "xrs_classify_moments_scratch_bytes": [ctypes.POINTER(I64)],
        "xrs_classify_moments": [P, I, I64, I64, I64, D, P, P, I64, P],
        "xrs_classify_select_scratch_bytes": [ctypes.POINTER(I64)],
        "xrs_classify_select": [I, P, I, I64, I64, I64, I, ctypes.c_uint64, P, I, P, P, ctypes.POINTER(I64), P, P,
                                I64, P],
        "xrs_classify_sort_scratch_bytes": [I64, I, ctypes.POINTER(I64)],
        "xrs_classify_sort": [P, I, I64, I64, I64, P, ctypes.POINTER(I64), P, I64, P],
        "xrs_classify_pick": [P, I, I64, I, ctypes.c_uint64, I64, P, I64, ctypes.POINTER(I64), P, P],
        "xrs_nb_sample_scratch_bytes": [I64, I64, ctypes.POINTER(I64)],
        "xrs_nb_sample": [I64, I64, ctypes.c_uint32, P, P, I64, ctypes.POINTER(I64), P],
        "xrs_nb_jenks_scratch_bytes": [I64, I, ctypes.POINTER(I64)],
        "xrs_nb_jenks": [P, I64, I, P, P, I64, P],
        "xrs_zonal_regions_scratch_bytes": [I64, I64, ctypes.POINTER(I64)],
        "xrs_zonal_regions": [P, I, I64, I64, I64, I, P, I64, P, I64, P],
        "xrs_zonal_bounds": [P, I, I64, I64, I64, I, P, P, I, P, P],
        "xrs_local_cells": [P, I64, P, I64, I64, I, I, P, I64, I, I, P, I64, P, I64, P, P],
        "xrs_local_combine_scratch_bytes": [I64, I64, ctypes.POINTER(I64)],
        "xrs_local_combine": [P, I64, P, I64, I64, I, P, I64, P, P, I64, P, P],
        "xrs_host_stencil":[I, P, I, P, I64, I64, P, P, I, P, I],
        "xrs_host_release": [I],
        "xrs_host_alloc": [ctypes.POINTER(P), I64],
        "xrs_host_free": [P],
        "xrs_synth_terrain_f32": [P, I64, I64, I64, I64, I64, ctypes.c_uint64, ctypes.c_float,
                                  ctypes.c_float, P],
        "xrs_debug_last_used_tma": [],
        "xrs_debug_last_grid": [],
        "xrs_debug_pick_seg_rows": [I64, I64, I64, I64, I64, I64, I64],
    }
    for name, args in sig.items():
        fn = getattr(lib, name)
        fn.argtypes = args
        fn.restype = I
    lib.xrs_last_error_string.argtypes = []
    lib.xrs_last_error_string.restype = ctypes.c_char_p
    lib.xrs_debug_pick_seg_rows.restype = I64
    return sig


EXPORTS = None


def lib():
    """Load (once) and return the shared library; raises if it was not built."""
    global _lib, EXPORTS
    if _lib is None:
        if not os.path.exists(SO_PATH):
            raise XrsError(
                "libxrs_b200.so is missing (%s): build it with `python __graft_entry__.py` / "
                "`python xarray-spatial_b200/_build.py`; there is no CPU fallback" % SO_PATH)
        l = ctypes.CDLL(SO_PATH)
        EXPORTS = _declare(l)
        _lib = l
    return _lib


def check(rc):
    if rc == XRS_OK:
        return
    msg = lib().xrs_last_error_string().decode("utf-8", "replace")
    if rc == XRS_EINVAL:
        raise ValueError(msg)
    if rc == XRS_EUNSUPPORTED:
        raise NotImplementedError(msg)
    if rc == XRS_ENOMEM:
        raise MemoryError(msg)
    raise XrsError(msg)


def call(name, *args):
    check(getattr(lib(), name)(*args))

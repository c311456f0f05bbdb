"""xrspatial_b200 -- H100 (sm_90a) backend for the dense 2-D stencil hot path of xarray-spatial.

Same public names as `xrspatial` for that path (SURVEY.md section 8a); every operator runs in
hand-written CUDA kernels behind the C ABI of include/xrs_b200.h.  There is no CPU fallback.
"""
from . import _lib  # noqa: F401
from ._xr import DataArray, Dataset  # noqa: F401
from .analytics import summarize_terrain, surface_suite  # noqa: F401
from .aspect import aspect  # noqa: F401
from .classify import binary, box_plot, equal_interval, head_tail_breaks, maximum_breaks  # noqa: F401
from .classify import natural_breaks, percentiles, quantile, reclassify, std_mean  # noqa: F401
from .convolution import convolution_2d, convolve_2d  # noqa: F401
from .curvature import curvature  # noqa: F401
from .focal import apply as focal_apply  # noqa: F401
from .focal import focal_stats, hotspots, mean  # noqa: F401
from .hillshade import hillshade  # noqa: F401
from .proximity import allocation, direction, euclidean_distance, great_circle_distance  # noqa: F401
from .proximity import manhattan_distance, proximity  # noqa: F401
from .pathfinding import a_star_search  # noqa: F401
from .perlin import perlin  # noqa: F401
from .multispectral import arvi, ebbi, evi, gci, nbr, nbr2, ndmi, ndvi, savi, sipi  # noqa: F401
from .slope import slope  # noqa: F401
from .terrain import generate_terrain  # noqa: F401
from .viewshed import viewshed  # noqa: F401
from .zonal import crop, regions, suggest_zonal_canvas, trim  # noqa: F401
from .zonal import crosstab as zonal_crosstab  # noqa: F401
from .zonal import stats as zonal_stats  # noqa: F401

__version__ = "0.1.0"

/*
 * xrs_b200.h -- C ABI of libxrs_b200.so, the H100 (sm_90a) backend for the dense 2-D
 * stencil hot path of xarray-spatial.
 *
 * The reference has no FFI: its backend seam is the set of Python runner callables that
 * xrspatial.utils.ArrayTypeFunctionMapping (utils.py:117-143) selects by array type, e.g.
 * slope._run_cupy(data, cellsize_x, cellsize_y) (slope.py:145).  Each entry point below is
 * what a fifth, "b200" runner of that mapping binds through ctypes; the comment on every
 * function names the reference runner it replaces (file:line in the reference's xrspatial/).
 * INTEGRATION.md shows the reference-side stub.
 *
 * Conventions
 *  - plain C types only; rasters are row-major (H rows = y, W cols = x); pitches in BYTES.
 *  - `*_f32` device entry points take DEVICE pointers and a cudaStream_t (as void*), only
 *    enqueue work on that stream and never synchronise or allocate user-visible memory (the one
 *    exception, convolve / focal statistics over wide windows, is described at those functions).
 *  - `xrs_host_*` entry points take HOST pointers (pinned or pageable), run the same kernels
 *    through an internal pipelined H2D / compute / D2H stripe engine, and return when the
 *    result is in `out`.  They are what a numpy-backed DataArray call uses.
 *  - return value: 0 on success, negative xrs_status otherwise; xrs_last_error_string()
 *    describes the last failure on the calling thread.  Nothing throws across the ABI.
 *  - inputs are never modified.
 */
#ifndef XRS_B200_H
#define XRS_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define XRS_ABI_VERSION 3

typedef void *xrs_stream_t; /* cudaStream_t */

enum xrs_status {
    XRS_OK = 0,
    XRS_EINVAL = -1,       /* bad argument (shape, null pointer, even kernel, ...) */
    XRS_ECUDA = -2,        /* CUDA runtime / driver error */
    XRS_EUNSUPPORTED = -3, /* valid request this build cannot serve */
    XRS_ENOMEM = -4
};

/* focal statistic ids (focal.py:782-790 `_function_mapping`) */
enum xrs_focal_stat {
    XRS_STAT_MEAN = 0, XRS_STAT_SUM = 1, XRS_STAT_MIN = 2, XRS_STAT_MAX = 3,
    XRS_STAT_STD = 4, XRS_STAT_RANGE = 5, XRS_STAT_VAR = 6
};

/* cell types of raster arguments.  Two sets of them:
 *   the raster set, XRS_F32 .. XRS_U16 (codes 0-5): read by proximity, viewshed, a_star_search and classify;
 *   the zonal set, every code (0-10): read by xrs_zonal_regions and xrs_zonal_bounds.
 * A code outside an entry point's set returns XRS_EINVAL ("unknown cell type"); its input pitch must be a multiple
 * of the cell size and at least a row. */
enum xrs_dtype { XRS_F32 = 0, XRS_F64 = 1, XRS_I32 = 2, XRS_I64 = 3, XRS_I16 = 4, XRS_U16 = 5,
                 XRS_I8 = 6, XRS_U8 = 7, XRS_U32 = 8, XRS_U64 = 9, XRS_BOOL = 10 };

int xrs_abi_version(void);
const char *xrs_last_error_string(void);
/* device 0..n-1 properties the Python layer needs to size launches / report rooflines */
int xrs_device_count(int *n);
int xrs_device_sm_count(int device, int *sm_count);

/* ------------------------------------------------------------------ surface (3x3)
 * All: in/out float32, 1-cell NaN ring, NaN inputs propagate to their 3x3 neighbourhood. */

/* slope._run_cupy (slope.py:145-160) / `_cpu` (slope.py:56-76): Horn slope in degrees. */
int xrs_slope_f32(const float *in, int64_t in_pitch, float *out, int64_t out_pitch,
                  int64_t H, int64_t W, double cellsize_x, double cellsize_y, xrs_stream_t s);
/* aspect._run_cupy (aspect.py:139-147) / `_run_numpy` (aspect.py:56-90): compass degrees,
 * -1 on flats; follows the CPU path (no 359.999 clamp). */
int xrs_aspect_f32(const float *in, int64_t in_pitch, float *out, int64_t out_pitch,
                   int64_t H, int64_t W, xrs_stream_t s);
/* curvature._run_cupy (curvature.py:81-95) / `_cpu` (curvature.py:31-41). */
int xrs_curvature_f32(const float *in, int64_t in_pitch, float *out, int64_t out_pitch,
                      int64_t H, int64_t W, double cellsize, xrs_stream_t s);
/* hillshade._run_cupy (hillshade.py:78-100) / `_run_numpy` (hillshade.py:20-35);
 * output float32 as the reference's GPU path and docs promise. */
int xrs_hillshade_f32(const float *in, int64_t in_pitch, float *out, int64_t out_pitch,
                      int64_t H, int64_t W, double azimuth, double angle_altitude,
                      xrs_stream_t s);
/* analytics.summarize_terrain (analytics.py:84-86) fused: one read, up to four writes.
 * Any output pointer may be NULL (that product is skipped); all outputs share out_pitch. */
int xrs_surface_suite_f32(const float *in, int64_t in_pitch, float *slope_out,
                          float *aspect_out, float *curvature_out, float *hillshade_out,
                          int64_t out_pitch, int64_t H, int64_t W, double cellsize_x,
                          double cellsize_y, double azimuth, double angle_altitude,
                          xrs_stream_t s);

/* slope / aspect with method='geodesic' (slope._run_cupy_geodesic slope.py:176-195,
 * aspect._run_cupy_geodesic aspect.py:179-198; arithmetic of geodesic.py:40-231): elevation float32
 * or float64 (elev_dtype XRS_F32 / XRS_F64), latitude / longitude in degrees as DEVICE float64
 * arrays -- lat[H], lon[W] for a regular grid (latlon_2d = 0) or (H, W) contiguous arrays for a
 * curvilinear one (latlon_2d = 1); z_factor converts the elevation unit to metres.  float32
 * output: slope in degrees, or compass aspect (-1 on flats) when want_aspect != 0. */
int xrs_geodesic(const void *elev, int elev_dtype, int64_t elev_pitch, const double *lat,
                 const double *lon, int latlon_2d, float *out, int64_t out_pitch, int64_t H, int64_t W,
                 double z_factor, int want_aspect, xrs_stream_t s);

/* Direct ingestion (SURVEY.md 8f-4): slope / aspect / curvature / hillshade (op = XRS_OP_*) on a
 * raster of int16, uint16, int32 or float64 cells (in_dtype = XRS_I16 / XRS_U16 / XRS_I32 / XRS_F64),
 * converted to float32 in registers exactly like the reference's `.astype(np.float32)`
 * (slope.py:58,150) but without the extra pass.  p: slope {csx, csy}; curvature {cellsize};
 * hillshade {azimuth, altitude}.  Needs 16-byte aligned rows and W % 4 == 0, else
 * XRS_EUNSUPPORTED (cast and use the float32 entry points). */
int xrs_surface_typed(int op, const void *in, int in_dtype, int64_t in_pitch, float *out,
                      int64_t out_pitch, int64_t H, int64_t W, const double *p, xrs_stream_t s);

/* ------------------------------------------------------------------ focal / convolution */
/* focal._mean_cupy (focal.py:135-146) / `_mean_numpy` (focal.py:44-67): ONE pass of the 3x3
 * NaN-skipping mean with clamped windows; centre cells equal (NaN-aware) to one of
 * `excludes` (host array, n_ex <= 8) are copied through.  f32: float in/out (sums in f64);
 * f64: double in/out.  in and out must not alias. */
int xrs_focal_mean_f32(const float *in, int64_t in_pitch, float *out, int64_t out_pitch,
                       int64_t H, int64_t W, const double *excludes, int n_ex, xrs_stream_t s);
int xrs_focal_mean_f64(const double *in, int64_t in_pitch, double *out, int64_t out_pitch,
                       int64_t H, int64_t W, const double *excludes, int n_ex, xrs_stream_t s);
/* float32 in, float64 out: what focal.mean's `agg.data.astype(float)` (focal.py:257) yields for
 * a float32 raster, without a separate widening pass */
int xrs_focal_mean_f32_f64(const float *in, int64_t in_pitch, double *out, int64_t out_pitch,
                           int64_t H, int64_t W, const double *excludes, int n_ex,
                           xrs_stream_t s);
/* convolution._convolve_2d_cupy (convolution.py:368-374) / `_convolve_2d_numpy` (:285-313):
 * correlation with a host float64 kernel (kh, kw odd, 1 .. 2047); NaN ring of (kh/2, kw/2).  Windows of
 * more than 49 x 49 taps or more than 63 cells on a side run on the wide-window kernel, which copies the
 * weights into a buffer allocated and freed on `s` (reentrant across streams).  That copy is from pageable
 * host memory: a table too large for the driver's staging buffers (a 2047 x 2047 window's 33.5 MB of
 * weights) may hold the call until earlier work on `s` is done, and wide windows cannot be captured into a
 * CUDA graph. */
int xrs_convolve2d_f32(const float *in, int64_t in_pitch, float *out, int64_t out_pitch,
                       int64_t H, int64_t W, const double *kernel, int kh, int kw,
                       xrs_stream_t s);
/* focal._focal_stats_cupy (focal.py:757-779) with the CPU semantics of `_apply_numpy`
 * (focal.py:305-326) + reducers (:268-302): cells where kernel == 1 participate, NaN and
 * out-of-raster cells are skipped.  `stat` is an xrs_focal_stat.  XRS_STAT_MEAN over a kernel of all
 * ones (np.ones((kh, kw)), the reference's FocalApply benchmark; odd kh, kw <= 25) runs on the running-box
 * kernel in NaN-skipping mode, O(1) work per cell; windows up to 49 x 49 taps and 63 per side on the tiled
 * kernels; wider ones (odd kh, kw up to 2047) on the wide-window kernel, with the mask in a buffer allocated
 * and freed on `s`. */
int xrs_focal_stat_f32(const float *in, int64_t in_pitch, float *out, int64_t out_pitch,
                       int64_t H, int64_t W, const double *kernel, int kh, int kw, int stat,
                       xrs_stream_t s);
/* focal.focal_stats (focal.py:800-878: seven `apply` calls stacked by xr.concat) in one pass:
 * plane i of `out` (planes `plane_stride` bytes apart, rows `out_pitch` bytes apart) receives
 * statistic stats[i] (xrs_focal_stat ids, no duplicates, n_stats <= 7).  The tile is loaded
 * once and swept twice for all seven statistics; results are bit-identical to n_stats calls
 * of xrs_focal_stat_f32.  Windows beyond 49 x 49 taps or 63 per side (odd sides up to 2047) take the
 * fused wide-window kernel: one sweep for mean / sum / min / max / range, a second only for var / std. */
int xrs_focal_stats_multi_f32(const float *in, int64_t in_pitch, float *out, int64_t out_pitch,
                              int64_t plane_stride, int64_t H, int64_t W, const double *kernel,
                              int kh, int kw, const int *stats, int n_stats, xrs_stream_t s);

/* focal.hotspots (focal.py:1050-1125) = convolve_2d with kernel / kernel.sum(), then
 * z = (mean - global_mean) / global_std classified into {0, +-90, +-95, +-99} (int8).
 * xrs_global_stats_f32: partial3[0..2] (device) <- count, sum(v - pivot), sum((v - pivot)^2) over
 * the non-NaN cells, from which np.nanmean / np.nanstd follow.  (focal.py:881-937) */
int xrs_global_stats_f32(const float *values, int64_t n, double pivot, double *partial3,
                         xrs_stream_t s);
int xrs_hotspots_classify_f32(const float *mean, int64_t n, double global_mean, double global_std,
                              int8_t *out, xrs_stream_t s);

/* ------------------------------------------------------------------ multispectral
 * Elementwise over n contiguous float32 cells; out is NaN where the denominator is 0. */
/* multispectral._run_normalized_ratio_cupy (:862) -- ndvi, nbr, nbr2, ndmi */
int xrs_normalized_ratio_f32(const float *a, const float *b, float *out, int64_t n, xrs_stream_t s);
/* multispectral._savi_cupy (:912) */
int xrs_savi_f32(const float *nir, const float *red, double soil_factor, float *out, int64_t n,
                 xrs_stream_t s);
/* multispectral._evi_cupy (:210) */
int xrs_evi_f32(const float *nir, const float *red, const float *blue, double c1, double c2,
                double soil_factor, double gain, float *out, int64_t n, xrs_stream_t s);
/* multispectral._arvi_cupy (:65) */
int xrs_arvi_f32(const float *nir, const float *red, const float *blue, float *out, int64_t n,
                 xrs_stream_t s);
/* multispectral._gci_cupy (:378) */
int xrs_gci_f32(const float *nir, const float *green, float *out, int64_t n, xrs_stream_t s);
/* multispectral._sipi_cupy (:1052) */
int xrs_sipi_f32(const float *nir, const float *red, const float *blue, float *out, int64_t n,
                 xrs_stream_t s);
/* multispectral._ebbi_cupy (:1195) */
int xrs_ebbi_f32(const float *red, const float *swir, const float *tir, float *out, int64_t n,
                 xrs_stream_t s);

/* ------------------------------------------------------------------ zonal.stats
 * zonal._stats_cupy (zonal.py:335-419) / `_stats_numpy` (:280-332) replaced by one streaming group-by that
 * discovers the zone ids and accumulates per-zone partials; mean / std / var are finalised from them by the
 * caller, and partials from several devices combine with sum / min / max (NCCL AllReduce).  (Round 1 also
 * exported a lookup-table kernel for a given id list, xrs_zonal_partials(_ex): 0.24 of the HBM roofline,
 * slower than the group-by it specialised; removed -- the float64 second pass now runs on the group-by
 * kernel, xrs_zonal_hash_second_pass.)
 *
 * zones (zones_dtype: I32, I64, F32, F64) and values (values_dtype: F32, F64) are device arrays of n
 * cells; a cell contributes to its zone if its value is finite and != nodata (when has_nodata). */

/* The group-by: aggregation into an open-addressing hash table of `cap` slots (power of two >= 1024; device
 * arrays keys/count/s1/s2/vmin/vmax of `cap` entries).  keys[slot] is the zone id (int64 for integer zones, the
 * bit pattern of the float64 value for float zones; INT64_MIN = empty, so an int64 zone INT64_MIN is not
 * counted in the table -- packed[3] reports it), s1/s2 are sums of (v - pivot) and (v - pivot)^2.  Every finite
 * zone value present in the raster gets a slot, also when none of its cells is valid (count 0).  row_len is the
 * raster's row length (n = rows * row_len): the scan walks down 128-column strips so that runs of equal zone ids
 * stay long. */

/* The first pass, with no host round trip in the middle: samples the pivot on the device (median of 4096
 * strided samples, unless use_pivot_hint: row stripes must share one pivot), empties the table, accumulates,
 * then compacts the used slots into `packed` (device, 4 + 6 * max_out doubles):
 *   packed[0] = used slots, packed[1] = table overflowed (grow `cap` and retry), packed[2] = pivot,
 *   packed[3] = an int64 zone INT64_MIN (the empty key, not in the table) was met: compute it apart,
 *   then 6 rows of max_out: key bit patterns, count (int64 bit patterns), s1, s2, min, max, in any
 *   order.  Slots beyond max_out are dropped (packed[0] > max_out tells; read the table instead).
 * flags: 3 device ints of scratch.  Replaces the sort + per-zone reductions of zonal.py:280-332. */
int xrs_zonal_hash_run(const void *values, int values_dtype, const void *zones, int zones_dtype, int64_t n,
                       int64_t row_len, int has_nodata, double nodata, int use_pivot_hint, double pivot_hint,
                       int64_t *keys, int64_t *count, double *s1, double *s2, double *vmin, double *vmax, int cap,
                       double *packed, int max_out, int *flags, xrs_stream_t s);

/* Second pass (numpy's two-pass variance, zonal.py:75-76 `ndarray.std / var`): the same
 * streaming group-by over the table xrs_zonal_hash_run left behind -- `keys` as populated by the first pass,
 * read only -- with sums taken about `zone_pivots[slot]` (device, `cap` doubles: the zone's mean from the
 * first pass) instead of one global pivot, so that s2 / n - (s1 / n)^2 does not cancel.  count / s1 / s2 /
 * vmin / vmax: a second set of `cap`-entry accumulators (reset here); `packed` / `flags` as above
 * (packed[2] = 0).  values_dtype XRS_F32 or XRS_F64.  */
int xrs_zonal_hash_second_pass(const void *values, int values_dtype, const void *zones, int zones_dtype, int64_t n,
                               int64_t row_len, int has_nodata, double nodata, const int64_t *keys,
                               const double *zone_pivots, int64_t *count, double *s1, double *s2, double *vmin,
                               double *vmax, int cap, double *packed, int max_out, int *flags, xrs_stream_t s);

/* `majority` (zonal.py:56-68): counts (zone, value) pairs of float32 values / int32 zones into
 * a hash table (keys/count of `cap` entries, emptied here; *overflow (device int) is set when it holds
 * fewer slots than the raster has distinct pairs; key =
 * (zone << 32) | (float32 bits of the value ^ 0x7fc00000), -0.0 folded into +0.0; the XOR makes the
 * empty key INT64_MIN stand for (zone INT32_MIN, a NaN), a pair never counted).  The caller picks the most
 * frequent value per zone (smallest value on ties). */
int xrs_zonal_pair_count(const float *values, const int32_t *zones, int64_t n, int64_t row_len,
                         int has_nodata, double nodata, int64_t *keys, int64_t *count, int cap,
                         int *overflow, xrs_stream_t s);

/* ------------------------------------------------------------------ proximity
 * proximity / allocation / direction (proximity.py:401-647) as an exact nearest-target transform: every cell gets
 * the target nearest to it under the metric, the first in row-major order among equidistant ones (the reference's
 * GDAL-style sweep only approximates this; DESIGN.md section 4.7).  Rasters of H x W cells of in_dtype (the raster
 * set), rows in_pitch bytes apart; x[W] and y[H] are DEVICE float64 coordinates, each strictly ascending
 * or strictly descending (GREAT_CIRCLE: degrees of longitude / latitude within +-180 / +-90).
 * targets: NULL for the default rule (nonzero and finite cells), else a DEVICE array of n_targets float64
 * values sorted ascending without NaN (a cell is a target when its value, widened to float64, is one of them;
 * n_targets may be 0: no cell is).  float32 output, rows out_pitch bytes apart: the distance
 * (XRS_PROX_DISTANCE), the nearest target's value (XRS_PROX_ALLOCATION) or the compass direction to it
 * (XRS_PROX_DIRECTION, 0 on targets); NaN where there is no target or the float32 squared distance exceeds
 * max_distance^2.
 * scratch: a DEVICE buffer of at least xrs_proximity_scratch_bytes(H, W, band_rows) bytes (about 8 bytes per
 * cell); band_rows (0: the library's choice) splits the column pass into bands and does not change the result.
 * Enqueues on `s` only; a bad argument returns XRS_EINVAL before any CUDA call. */
enum xrs_metric { XRS_METRIC_EUCLIDEAN = 0, XRS_METRIC_GREAT_CIRCLE = 1, XRS_METRIC_MANHATTAN = 2 };
enum xrs_prox_mode { XRS_PROX_DISTANCE = 0, XRS_PROX_ALLOCATION = 1, XRS_PROX_DIRECTION = 2 };
int xrs_proximity_scratch_bytes(int64_t H, int64_t W, int band_rows, int64_t *bytes);
int xrs_proximity(const void *in, int in_dtype, int64_t in_pitch, int64_t H, int64_t W, const double *x,
                  const double *y, const double *targets, int n_targets, double max_distance, int metric,
                  int mode, float *out, int64_t out_pitch, void *scratch, int64_t scratch_bytes, int band_rows,
                  xrs_stream_t s);

/* ------------------------------------------------------------------ viewshed
 * viewshed (viewshed.py:1122-1502) as a per-cell line-of-sight test that makes the reference sweep's
 * visible / invisible decision (DESIGN.md section 4.8).  Rasters of H x W cells of in_dtype (the raster set,
 * read as float64, never written), rows in_pitch bytes apart; the observer stands on cell (vp_row, vp_col) at
 * vp_elev; target_elev is added to every cell seen as a target; ew_res / ns_res are the coordinate steps between
 * columns / rows (may be negative or NaN).  float64 output, rows out_pitch bytes apart: 180 at the observer, the
 * vertical angle in degrees of a visible cell, -1 otherwise (NaN cells never block and are -1).
 * scratch: a DEVICE buffer of at least xrs_viewshed_scratch_bytes(H, W) bytes (56 bytes per cell).
 * Enqueues on `s` only; a bad argument returns XRS_EINVAL before any CUDA call. */
int xrs_viewshed_scratch_bytes(int64_t H, int64_t W, int64_t *bytes);
int xrs_viewshed(const void *in, int in_dtype, int64_t in_pitch, int64_t H, int64_t W, int64_t vp_row,
                 int64_t vp_col, double vp_elev, double target_elev, double ew_res, double ns_res, double *out,
                 int64_t out_pitch, void *scratch, int64_t scratch_bytes, xrs_stream_t s);

/* ------------------------------------------------------------------ a_star_search
 * a_star_search (pathfinding.py:233-382) as an exact shortest-path search (DESIGN.md section 4.9).  Rasters of
 * H x W cells of in_dtype (the raster set, read as float64, never written), rows in_pitch bytes apart, H W < 2^31.
 * A cell is crossable unless it is NaN or equal to one of the n_barriers DEVICE float64 values in `barriers`
 * (NULL when n_barriers is 0).  Moves go to the 8 neighbours, or 4 with connectivity 4, and cost 1 or sqrt(2).
 * xrs_a_star_search: float64 output, rows out_pitch bytes apart, NaN except along a shortest path from the start
 * to the goal, which holds the running sum of the step lengths (0 at the start); all NaN when there is no path.
 * Among equally short paths it takes, from each cell, the first move of the reference's neighbour order that stays
 * on a shortest path.  *rounds (may be NULL) receives the number of relaxation rounds.  scratch: a DEVICE buffer
 * of at least xrs_a_star_scratch_bytes(H, W) bytes (about 9 bytes per cell); after the call it holds, from byte
 * 256, the field of shortest lengths to the goal as int32 pairs (orthogonal, diagonal steps; INT32_MAX, 0 where
 * no path reaches), row-major.
 * xrs_a_star_snap: the cell _find_nearest_pixel picks for (row, col): itself when crossable, else the crossable
 * cell at the least pixel distance below the raster's diagonal, the first in row-major order among equals; -1, -1
 * when there is none.  scratch: a DEVICE buffer of at least 256 bytes.
 * Unlike the other entry points, both SYNCHRONIZE with `s` before they return: the search reads an activity
 * count every few rounds and the snap returns its cell.  A bad argument returns XRS_EINVAL before any CUDA call. */
int xrs_a_star_scratch_bytes(int64_t H, int64_t W, int64_t *bytes);
int xrs_a_star_search(const void *in, int in_dtype, int64_t in_pitch, int64_t H, int64_t W, const double *barriers,
                      int n_barriers, int connectivity, int64_t start_row, int64_t start_col, int64_t goal_row,
                      int64_t goal_col, double *out, int64_t out_pitch, void *scratch, int64_t scratch_bytes,
                      int64_t *rounds, xrs_stream_t s);
int xrs_a_star_snap(const void *in, int in_dtype, int64_t in_pitch, int64_t H, int64_t W, const double *barriers,
                    int n_barriers, int64_t row, int64_t col, int64_t *snap_row, int64_t *snap_col, void *scratch,
                    int64_t scratch_bytes, xrs_stream_t s);

/* ------------------------------------------------------------------ perlin / generate_terrain
 * perlin (perlin.py:189) and generate_terrain (terrain.py:183) with the reference's NumPy path as the semantics
 * (DESIGN.md section 4.10).
 * xrs_perm_tables: for each of the n_seeds (1 .. 32) HOST seeds, writes RandomState(seed).permutation(n) as int32
 * to `tables` (DEVICE, n_seeds x n, n 1 .. 2^20), bit for bit.  scratch: a DEVICE buffer of at least
 * xrs_perm_tables_scratch_bytes(n_seeds, n) bytes (about 22 bytes per table entry plus 2 MB per seed).  *rounds
 * (may be NULL) receives the number of reservation rounds of the shuffle.  It SYNCHRONIZES with `s`: the host reads
 * how far the draws got and how many steps are pending between batches of launches.
 * xrs_noise: H x W cells of float32 or float64 (dtype), rows in_pitch / out_pitch bytes apart; `in` (read only for
 * terrain, never written) and `out` have the same cell type.  terrain 0 is perlin: one octave from tables[0 .. 2^20)
 * at the float32 DEVICE coordinates xs (W values) and ys (H values), then (d - min) / (max - min).  terrain 1 is
 * generate_terrain: 16 octaves, octave o from tables[o 2^20 ..) at float32(x 2^o) weighed by 2^-o, added to in 0,
 * then / 1.97, the cube, the same normalisation, cells below 0.3 set to 0, and the product with zfactor.
 * index_stats (DEVICE, 5 int32 per octave: a bad-coordinate flag, the least and largest of P[xi] and P[xi + 1] over
 * the columns, the least and largest yi over the rows) tells the caller whether the reference would index its
 * doubled table outside [-2^21, 2^21) and raise IndexError; the output is then meaningless.  scratch: a DEVICE
 * buffer of at least xrs_noise_scratch_bytes(H, W, terrain) bytes (24 bytes per row and column per octave); after
 * the call its first 16 bytes hold the field's min and max before normalisation, as float64.  Enqueue-only.  A bad argument returns
 * XRS_EINVAL before any CUDA call. */
int xrs_perm_tables_scratch_bytes(int n_seeds, int64_t n, int64_t *bytes);
int xrs_perm_tables(const uint32_t *seeds, int n_seeds, int64_t n, int32_t *tables, void *scratch,
                    int64_t scratch_bytes, int64_t *rounds, xrs_stream_t s);
int xrs_noise_scratch_bytes(int64_t H, int64_t W, int terrain, int64_t *bytes);
int xrs_noise(const void *in, int dtype, int64_t in_pitch, int64_t H, int64_t W, const int32_t *tables,
              const float *xs, const float *ys, int terrain, double zfactor, void *out, int64_t out_pitch,
              int32_t *index_stats, void *scratch, int64_t scratch_bytes, xrs_stream_t s);

/* ------------------------------------------------------------------ classify (classify.cu)
 * Rasters are H x W cells of `dtype` (the raster set), rows in_pitch bytes apart, read and never written.  A key is
 * the order-preserving unsigned image of a cell's bits (-0.0 folded into +0.0; 16-, 32- or 64-bit by the cell
 * type); "finite" is every integer cell and the float cells that are neither NaN nor +-inf.
 * xrs_classify_cells: member 0 is the reference's _cpu_bin: each finite cell is compared in float64 with bins[nb]
 * (DEVICE) by its binary search and gets new_values[bin] (DEVICE float32), anything else NaN; float32 out.  member
 * 1 is _cpu_binary: 1 where the cell equals one of the nb DEVICE float64 values, else 0 (NaN for a non-finite
 * float cell); out has the cell type.  nb = 0 is allowed.  Enqueue-only.
 * xrs_classify_moments: out5 (DEVICE float64) = count, mean, M2 (sum of squared deviations), min and max of the
 * finite cells above `above` (-inf: all of them), each CTA merging in a fixed order.  Enqueue-only.
 * xrs_classify_select: exact order statistics by 8-bit digit passes from the top of a `bits`-wide key; each pass
 * reads the source once for every rank.  source 0: the raster's finite cells.  source 1: the gaps of the unique
 * values of xrs_classify_sort's keys (in: those keys, H = 1, W = their count; the gap at position i is the cell
 * type's difference of keys i and i - 1 when they differ).  source 2: the positions of the gaps whose key is `tie`.
 * With nr = 0 it runs the top-digit pass, writes its 256 counts to hist0 (HOST) and the number of keys to
 * *n_keys; with nr > 0, hist0 must hold those counts, and keys[i] (HOST) gets the ranks[i]-th smallest key
 * (0-based, HOST ranks) and rem[i] the rank less the keys below that key.  SYNCHRONIZES with `s` every pass.
 * xrs_classify_sort: the finite cells' keys, sorted ascending by an LSD radix sort, into keys (DEVICE, n_keys
 * entries of 4 bytes, or 8 for 64-bit keys; room for H W).  SYNCHRONIZES with `s` once, to read the count.
 * xrs_classify_pick: over n sorted keys, mode 0 writes every unique key (in no order), mode 1 the key pairs
 * (i - 1, i) of the gaps above key `tie` or equal to it at a position >= pos; at most cap entries (pairs) go to
 * out (DEVICE), *count gets how many there are.  scratch: 8 bytes.  SYNCHRONIZES with `s`.
 * A bad argument returns XRS_EINVAL before any CUDA call. */
int xrs_classify_cells(const void *in, int dtype, int64_t in_pitch, int64_t H, int64_t W, int member,
                       const double *bins, const float *new_values, int nb, void *out, int64_t out_pitch,
                       xrs_stream_t s);
int xrs_classify_moments_scratch_bytes(int64_t *bytes);
int xrs_classify_moments(const void *in, int dtype, int64_t in_pitch, int64_t H, int64_t W, double above,
                         double *out5, void *scratch, int64_t scratch_bytes, xrs_stream_t s);
int xrs_classify_select_scratch_bytes(int64_t *bytes);
int xrs_classify_select(int source, const void *in, int dtype, int64_t in_pitch, int64_t H, int64_t W, int bits,
                        uint64_t tie, const int64_t *ranks, int nr, uint64_t *keys, int64_t *rem, int64_t *n_keys,
                        uint64_t *hist0, void *scratch, int64_t scratch_bytes, xrs_stream_t s);
int xrs_classify_sort_scratch_bytes(int64_t n, int dtype, int64_t *bytes);
int xrs_classify_sort(const void *in, int dtype, int64_t in_pitch, int64_t H, int64_t W, void *keys, int64_t *n_keys,
                      void *scratch, int64_t scratch_bytes, xrs_stream_t s);
int xrs_classify_pick(const void *sorted, int dtype, int64_t n, int mode, uint64_t tie, int64_t pos, void *out,
                      int64_t cap, int64_t *count, void *scratch, xrs_stream_t s);

/* ------------------------------------------------------------------ natural_breaks (natural_breaks.cu)
 * xrs_nb_sample: the set of the first s entries of np.linspace(0, n, n, dtype=uint32) after
 * RandomState(seed).shuffle -- the reference's sample of cell indices -- in ascending order, as int64 to out
 * (DEVICE, s entries), for 1 <= s < n <= 2^32 (more cells: XRS_EINVAL).  scratch: a DEVICE buffer of at least
 * xrs_nb_sample_scratch_bytes(n, s) bytes (about 10 bytes per cell).  *rounds (may be NULL) receives how many
 * rounds the chunked resolve took to settle.  It SYNCHRONIZES with `s` once per round.
 * xrs_nb_jenks: the reference's _run_numpy_jenks_matrices over the n sorted float32 DEVICE values x for k classes:
 * lower_class_limits to lcl (DEVICE float32, (k + 1) x (n + 1), column j at j (n + 1)) and var_combinations, laid
 * out the same way, at the start of scratch (DEVICE, xrs_nb_jenks_scratch_bytes(n, k) bytes), bit for bit.
 * (k - 1) n^2 / 2 iterations on top of the first column's n^2 / 2.  Enqueue-only.
 * A bad argument returns XRS_EINVAL before any CUDA call. */
int xrs_nb_sample_scratch_bytes(int64_t n, int64_t s, int64_t *bytes);
int xrs_nb_sample(int64_t n, int64_t s, uint32_t seed, int64_t *out, void *scratch, int64_t scratch_bytes,
                  int64_t *rounds, xrs_stream_t stream);
int xrs_nb_jenks_scratch_bytes(int64_t n, int k, int64_t *bytes);
int xrs_nb_jenks(const float *x, int64_t n, int k, float *lcl, void *scratch, int64_t scratch_bytes,
                 xrs_stream_t stream);

/* ------------------------------------------------------------------ zonal regions / trim / crop (zonal_regions.cu)
 * Rasters of H x W cells of `dtype` (the zonal set), rows in_pitch bytes apart, H and W below 2^31, read and never
 * written.
 * xrs_zonal_regions: zonal.regions (zonal.py:1406-1549): the reference's label of every cell for the 4- or 8-cell
 * neighbourhood, as int64 cast once to the cell type (bool: all true), NaN for NaN cells, to out (DEVICE, the cell
 * type, rows out_pitch bytes apart).  scratch: a DEVICE buffer of at least xrs_zonal_regions_scratch_bytes(H, W)
 * bytes (10 bytes per cell below 2^31 cells, 18 above).  Enqueue-only.
 * xrs_zonal_bounds: the least and largest row, then the least and largest column, of the cells that equal none of
 * the n_values values (mode 0, zonal.trim) or one of them (mode 1, zonal.crop), as int64 to out4 (DEVICE); rows
 * LLONG_MAX, -1 and columns LLONG_MAX, -1 when no cell qualifies.  values (DEVICE float64) holds the values;
 * int_values (DEVICE int64, or NULL when any value is not an integer) holds them again as integers, and integer
 * cells other than uint64 then compare exactly; everything else compares in float64, where NaN equals nothing.
 * Enqueue-only.
 * A bad argument returns XRS_EINVAL before any CUDA call. */
int xrs_zonal_regions_scratch_bytes(int64_t H, int64_t W, int64_t *bytes);
int xrs_zonal_regions(const void *in, int dtype, int64_t in_pitch, int64_t H, int64_t W, int neighborhood, void *out,
                      int64_t out_pitch, void *scratch, int64_t scratch_bytes, xrs_stream_t s);
int xrs_zonal_bounds(const void *in, int dtype, int64_t in_pitch, int64_t H, int64_t W, int mode,
                     const double *values, const int64_t *int_values, int n_values, int64_t *out4, xrs_stream_t s);

/* ------------------------------------------------------------------ host-buffer (end-to-end)
 * Same operators on HOST rasters: the library cuts the raster into row chunks and overlaps
 * host->device copies, kernels and device->host copies on internal streams.  `op` selects
 * the operator (values 0-3 are also the `op` of xrs_surface_typed). */
enum xrs_op {
    XRS_OP_SLOPE = 0, XRS_OP_ASPECT = 1, XRS_OP_CURVATURE = 2, XRS_OP_HILLSHADE = 3,
    XRS_OP_FOCAL_MEAN = 4, XRS_OP_CONVOLVE = 5, XRS_OP_FOCAL_STAT = 6
};
/* in: H x W cells of `in_dtype`, out: H x W cells, both contiguous rows in host memory:
 *   slope, aspect, curvature, hillshade: float32 in, or int16 / uint16 / int32 / float64 when
 *     W % 4 == 0 (xrs_surface_typed behind the pipeline: the raw cells cross PCIe); float32 out.
 *   focal mean: float32 or float64 in; float64 out (focal.py:257 `astype(float)`).
 *   convolve, focal stat: float32 in, float32 out.
 * p: slope {csx, csy}; curvature {cellsize}; hillshade {azimuth, altitude};
 *    convolve {kh, kw}; focal stat {kh, kw, stat}.  aux/naux (host): the excludes of focal mean,
 *    or the kernel of convolve / focal stat.
 * devices: CUDA ordinals, each at most once.  The output rows are cut into one stripe per listed
 * device, each stripe runs the chunk pipeline on its own host thread and PCIe link; the halo rows
 * of a stripe come from the host raster, so there is no device-to-device traffic.  This is the
 * reference's dask.map_overlap(depth=r, boundary=nan) over row blocks (slope.py:94-97,
 * focal.py:72-75) for host rasters.  A bad request returns XRS_EINVAL before any CUDA call. */
int xrs_host_stencil(int op, const void *in, int in_dtype, void *out, int64_t H, int64_t W,
                     const double *p, const double *aux, int naux, const int *devices, int n_devices);
/* frees the per-device staging buffers the host path keeps between calls */
int xrs_host_release(int device);
/* pinned host memory helpers (cudaHostAlloc / cudaFreeHost) for callers that want
 * full-speed DMA on the host path */
int xrs_host_alloc(void **ptr, int64_t bytes);
int xrs_host_free(void *ptr);

/* test / profiling hooks: which kernel the last launch on this thread chose -- 0 cp.async strip
 * kernel, 1 TMA strip kernel, 2 direct-ingest TMA kernel, 3 running-box kernel (uniform convolve_2d, focal.apply
 * mean over an all-ones window), 4 generic tiled convolve, 5 bounds-checked convolve fallback, 6 fused focal
 * statistics, 7 tiled single focal statistic, 8 bounds-checked focal statistic fallback, 9 zonal group-by
 * (xrs_zonal_hash_run / _second_pass), 10 zonal pair count (xrs_zonal_pair_count), 11 wide-window convolve,
 * 12 wide-window single focal statistic, 13 wide-window fused focal statistics, 14 proximity row pass, 15 classify per-cell pass -- and with how many CTAs */
int xrs_debug_last_used_tma(void);
int xrs_debug_last_grid(void);
/* host-only test hook: the row-segment height the persistent kernels pick for a raster of H rows cut into
 * n_tiles column tiles, dealt round-robin to `resident` CTAs (at least min_rows, rows + lead a multiple of
 * quantum, about `want` tasks per CTA): minimises ceil(tasks / resident) x (rows + lead). */
int64_t xrs_debug_pick_seg_rows(int64_t H, int64_t n_tiles, int64_t resident, int64_t min_rows, int64_t lead,
                                int64_t quantum, int64_t want);

/* ------------------------------------------------------------------ synthetic inputs
 * Deterministic fBm-like terrain (value-noise octaves), a pure function of
 * (seed, global row, global col): stripes generated on different devices tile exactly.
 * Used by bench.py and the tests; not part of the reference API. */
int xrs_synth_terrain_f32(float *out, int64_t out_pitch, int64_t H, int64_t W,
                          int64_t row0, int64_t col0, uint64_t seed, float zmin, float zmax,
                          xrs_stream_t s);

#ifdef __cplusplus
}
#endif
#endif /* XRS_B200_H */

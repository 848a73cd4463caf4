/* wb2b200.h -- C ABI of the H100-native WeatherBench2 hot path (libwb2b200.so).
 *
 * The reference (google-research/weatherbench2) is pure Python and has no FFI of
 * its own; these entry points are what its operator classes bind through
 * ctypes (see INTEGRATION.md).  Each entry point cites the reference interface
 * it replaces (paths relative to the reference checkout).
 *
 * Conventions
 *   - every function returns 0 on success, a negative WB2_E* code on failure and
 *     never throws/aborts; wb2_last_error() gives the message (thread-local);
 *   - the caller owns every data buffer.  "dev" pointers are CUDA device
 *     pointers on the context's device, "host" pointers are ordinary host
 *     memory (pinned or pageable);  small descriptor arrays (weights, offset
 *     tables) are ALWAYS host pointers and are copied by the library;
 *   - kernels are enqueued on the context's stream; results written to device
 *     memory are ordered on that stream (wb2_synchronize / wb2_memcpy_d2h to
 *     read them);  the *_host entry points are synchronous end to end;
 *   - outputs are raw weighted SUMS (and weight sums) in float64; division,
 *     sqrt, ACC ratio, CRPS = skill - spread/2 stay in the Python operator so
 *     the NaN / zero-weight rules remain visible (weatherbench2/metrics.py:161);
 *   - reductions are deterministic (fixed-order tree, no float atomics).
 *
 * Field addressing.  A "field" is one 2-D (row, col) slab with `col`
 * contiguous: (latitude, longitude) for raw 0.25-degree data or
 * (longitude, latitude) for the reference's mock / regridded layout
 * (weatherbench2/schema.py:83).  Operands are addressed by a base pointer plus
 * a per-field element-offset table, so broadcasting (truth without lead_time),
 * the by-init gather `truth.sel(time=valid_time)` (evaluation.py:475) and the
 * climatology day-of-year lookup (metrics.py:398-404) need no materialised
 * copies.
 */
#ifndef WB2B200_H_
#define WB2B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define WB2_VERSION 100 /* 0.1.0 */

enum {
  WB2_OK = 0,
  WB2_EINVAL = -1,   /* bad argument */
  WB2_ECUDA = -2,    /* CUDA runtime error (message has the cudaError string) */
  WB2_ENOMEM = -3,
  WB2_EUNSUPPORTED = -4
};

enum { WB2_F32 = 0, WB2_F64 = 1 };

#define WB2_MAX_REGIONS 32

/* number of per-(field, region) float64 outputs of wb2_det_metrics */
#define WB2_DET_NSTAT 10
/* [0] sum W*d^2   [1] sum W*|d|   [2] sum W*d          (d  = f - t)
 * [3] sum W*fa*ta [4] sum W*fa^2  [5] sum W*ta^2       (fa = f - c, ta = t - c)
 * [6] sum W*[d valid] [7] sum W*[fa*ta valid] [8] sum W*[fa valid]
 * [9] sum W*[ta valid]   -- the xarray `sum_of_weights` of each average     */

/* number of per-(field, region) float64 outputs of wb2_ens_metrics */
#define WB2_ENS_NSTAT 10
/* [0] sum W*skill_pt      skill_pt  = mean_m |t - x_m|        (metrics.py:824)
 * [1] sum W*spread_pt     spread_pt = 2 mean_m((2r_m-M-1)x_m)/(M-1)  (:805-813)
 * [2] sum W*(t - xbar)^2                                       (metrics.py:1330)
 * [3] sum W*var_ddof1                                          (metrics.py:1238)
 * [4] sum W*((t - xbar)^2 - var/M)                             (metrics.py:564-565)
 * [5..9] the matching sums of W*[value valid]                                */

typedef struct wb2_ctx wb2_ctx;

/* Region / latitude weights of one launch.  The weight of cell (row, col) for
 * region r is   W_r = row_w[r][row] * seg_w[r][seg(col)] * col_w[col] * cell_w[row][col]
 * where seg(col) = k for seg_start[k] <= col < seg_start[k+1].
 * This factorisation holds every reference region exactly
 * (weatherbench2/regions.py:57-158): latitude weights and latitude boxes go in
 * row_w (or col_w*seg_w for the latitude-fastest layout), longitude boxes in
 * seg_w (or row_w), a LandRegion mask in cell_w.
 * zero_skip != 0 reproduces `dataset.where(weights > 0, 0)` (metrics.py:160):
 * cells whose weight is zero contribute nothing, even when they hold NaN/Inf.
 * It requires non-negative weights: a negative row_w / seg_w / col_w entry is
 * rejected with WB2_EINVAL (cell_w, a device array, is not checked; it must be
 * non-negative too).  With zero_skip == 0 any sign is accepted and the sums
 * are linear in W.                                                          */
typedef struct {
  int32_t nrow;            /* slow spatial axis length                         */
  int32_t ncol;            /* contiguous spatial axis length                   */
  int64_t row_stride;      /* elements between consecutive rows (>= ncol)      */
  int32_t nregion;         /* 1..WB2_MAX_REGIONS                               */
  int32_t nseg;            /* >= 1                                             */
  const double* row_w;     /* host [nregion][nrow]                             */
  const int32_t* seg_start;/* host [nseg + 1], seg_start[0]=0, [nseg]=ncol     */
  const double* seg_w;     /* host [nregion][nseg]                             */
  const float* col_w;      /* host [ncol] or NULL (== all ones)                */
  const float* cell_w;     /* DEVICE [nrow][ncol] (dense) or NULL              */
  int32_t zero_skip;
} wb2_weights;

/* ---- library / context ---------------------------------------------------- */
int wb2_version(void);
const char* wb2_last_error(void);
/* 1 when the library was built with the CUDA kernels (always, for this .so)   */
int wb2_has_cuda(void);
/* number of kernels this context has launched since creation (bench evidence) */
int64_t wb2_launch_count(const wb2_ctx* ctx);

int wb2_create(int device, wb2_ctx** out);
int wb2_destroy(wb2_ctx* ctx);
/* use an external cudaStream_t (e.g. torch's current stream); NULL = own stream */
int wb2_set_stream(wb2_ctx* ctx, void* cuda_stream);
void* wb2_get_stream(wb2_ctx* ctx);
int wb2_synchronize(wb2_ctx* ctx);
/* Ordering with a caller-owned stream WITHOUT blocking the host (the context's
 * own stream is cudaStreamNonBlocking, so nothing orders it implicitly against
 * e.g. torch's current stream):
 *   wb2_wait_stream : work enqueued on the context AFTER this call waits for
 *                     everything already enqueued on `cuda_stream` (inputs
 *                     still being produced there);
 *   wb2_stream_wait : work enqueued on `cuda_stream` AFTER this call waits for
 *                     everything already enqueued on the context (results).
 * No-ops when `cuda_stream` is the context's stream (wb2_set_stream).  NULL is
 * the legacy default stream.                                                  */
int wb2_wait_stream(wb2_ctx* ctx, void* cuda_stream);
int wb2_stream_wait(wb2_ctx* ctx, void* cuda_stream);

int wb2_malloc(wb2_ctx* ctx, size_t bytes, void** dev_ptr);
int wb2_free(wb2_ctx* ctx, void* dev_ptr);
int wb2_host_alloc(wb2_ctx* ctx, size_t bytes, void** host_ptr); /* pinned */
int wb2_host_free(wb2_ctx* ctx, void* host_ptr);
int wb2_memcpy_h2d(wb2_ctx* ctx, void* dev_dst, const void* host_src, size_t bytes);
int wb2_memcpy_d2h(wb2_ctx* ctx, void* host_dst, const void* dev_src, size_t bytes);
int wb2_memset(wb2_ctx* ctx, void* dev_ptr, int value, size_t bytes);

/* ---- K1: deterministic metrics ---------------------------------------------
 * Replaces the arithmetic of  MSE / RMSESqrtBeforeTimeAvg / MAE / Bias / ACC
 * .compute_chunk (weatherbench2/metrics.py:251-269, 283-301, 323-330, 352-359,
 * 387-414) and of _spatial_average (metrics.py:141-163) for ALL regions of an
 * eval config in one pass over the data (evaluation.py:408-435 loops
 * metric x region and re-reads the chunk every time).
 *   f, t, c      device base pointers (c may be NULL: no climatology -> stats
 *                3,4,5,7,8,9 are written as 0)
 *   dtype        WB2_F32 / WB2_F64 element type of f, t and c
 *   off_f/t/c    host [nfield] element offsets of each field's slab
 *   skipna       0: NaN propagates into the sums (stats 6..9 then hold the
 *                plain weight sums);  1: NaN cells are skipped per statistic
 *   out          device [nfield][nregion][WB2_DET_NSTAT] float64
 */
int wb2_det_metrics(wb2_ctx* ctx, const void* f, const void* t, const void* c,
                    int dtype, int64_t nfield, const int64_t* off_f,
                    const int64_t* off_t, const int64_t* off_c,
                    const wb2_weights* w, int skipna, double* out);

/* Wind-vector variant: stat[0] = sum W*(du^2 + dv^2), stat[6] its weight sum
 * (WindVectorMSE.compute_chunk, metrics.py:189-202); other stats are 0.       */
int wb2_det_metrics_vector(wb2_ctx* ctx, const void* fu, const void* fv,
                           const void* tu, const void* tv, int dtype,
                           int64_t nfield, const int64_t* off_fu,
                           const int64_t* off_fv, const int64_t* off_tu,
                           const int64_t* off_tv, const wb2_weights* w,
                           int skipna, double* out);

/* Same as wb2_det_metrics but f, t, c are HOST base pointers and `out` is a
 * host array: the library streams the slabs through double-buffered device
 * staging (H2D on a copy stream overlapped with the kernel) and returns after
 * the result is in `out`.  This is the end-to-end entry the Python operators
 * use for NumPy inputs.  cell_w in `w` must still be a device pointer.        */
int wb2_det_metrics_host(wb2_ctx* ctx, const void* f, const void* t,
                         const void* c, int dtype, int64_t nfield,
                         const int64_t* off_f, const int64_t* off_t,
                         const int64_t* off_c, const wb2_weights* w, int skipna,
                         double* out_host);

/* ---- host-streaming entries and the slab cache ----------------------------------
 * Every *_host entry takes HOST base pointers (pinned memory reaches the PCIe
 * rate; pageable memory works at the driver's staging rate), streams the 2-D
 * slabs through two device staging buffers with the copies overlapped against
 * the kernels, and returns after the result is in host memory.
 *
 * wb2_set_slab_cache(ctx, bytes) reserves `bytes` of HBM as an LRU cache of
 * host slabs keyed by host address: the operands that repeat from chunk to
 * chunk -- the truth slabs of truth.sel(time=valid_time) (evaluation.py:475)
 * and the climatology slabs of the day-of-year lookup (metrics.py:398-404) --
 * then cross PCIe once instead of once per chunk (the forecast is never
 * cached).  The caller must not modify cached host arrays while the cache is
 * enabled; bytes = 0 (the default) disables it and frees the arena.
 * wb2_transfer_stats: which = 0 H2D bytes, 1 D2H bytes, 2 cache hits,
 * 3 cache misses of the *_host entries since the last reset.                     */
int wb2_set_slab_cache(wb2_ctx* ctx, size_t bytes);
int64_t wb2_transfer_stats(const wb2_ctx* ctx, int which);
int wb2_reset_transfer_stats(wb2_ctx* ctx);

/* wb2_ens_metrics on host buffers (x, t host base pointers, out host
 * [nfield][nregion][WB2_ENS_NSTAT]); truth slabs go through the slab cache.      */
int wb2_ens_metrics_host(wb2_ctx* ctx, const void* x, const void* t, int dtype,
                         int32_t nmember, int64_t member_stride, int64_t nfield,
                         const int64_t* off_x, const int64_t* off_t,
                         const wb2_weights* w, int skipna, double* out_host);

/* ---- K2: ensemble metrics --------------------------------------------------
 * Replaces CRPS / CRPSSkill / CRPSSpread, EnsembleMeanMSE / RMSE,
 * EnsembleVariance / Stddev, DebiasedEnsembleMeanMSE .compute_chunk
 * (metrics.py:657-715, 1185-1241, 1293-1363) incl. _rankdata (:836-846):
 * all five point-wise quantities from ONE read of the M members.
 *   x            device base pointer of the ensemble forecast
 *   off_x        host [nfield] offset of member 0 of each field
 *   member_stride elements between consecutive members of the same cell
 *   t, off_t     truth slab per field
 *   out          device [nfield][nregion][WB2_ENS_NSTAT] float64
 * 1..64 members: register sorting networks (the fast path); 65..1551 members
 * (metrics_test.py uses 100 and 1000): rank by counting in shared memory;
 * more: WB2_EUNSUPPORTED.
 */
int wb2_ens_metrics(wb2_ctx* ctx, const void* x, const void* t, int dtype,
                    int32_t nmember, int64_t member_stride, int64_t nfield,
                    const int64_t* off_x, const int64_t* off_t,
                    const wb2_weights* w, int skipna, double* out);

/* ---- K3: energy score -------------------------------------------------------
 * Replaces the per-member weighted L2 norms of EnergyScoreSkill / Spread
 * (metrics.py:1471-1517): every member is read once.
 *   out   device [nfield][nregion][4][nmember] float64:
 *         [0][m] sum W (x_m - t)^2         [1][m] sum W (x_m - x_{m+1})^2 (m < M-1)
 *         [2][m], [3][m] the matching weight sums
 * NaN propagates (skipna = False semantics); 1..64 members.                     */
int wb2_energy_score(wb2_ctx* ctx, const void* x, const void* t, int dtype,
                     int32_t nmember, int64_t member_stride, int64_t nfield,
                     const int64_t* off_x, const int64_t* off_t,
                     const wb2_weights* w, double* out);

/* ---- K6: map-output ("Spatial*") metrics with the time mean fused in ---------
 * Replaces SpatialBias / SpatialMSE / SpatialMAE .compute_chunk
 * (metrics.py:304-374) and the `.mean(time, skipna)` of Metric.compute
 * (metrics.py:117-138): out[j] = mean_g stat(f[j*ngroup+g], t[j*ngroup+g]) per
 * grid cell.  ngroup == 1 gives the per-time maps of compute_chunk unchanged.
 *   stat        WB2_MAP_BIAS f - t | WB2_MAP_MSE (f - t)^2 | WB2_MAP_MAE |f - t|
 *   off_f/off_t host [nout * ngroup] element offsets of the slabs (group-major)
 *   nrow, ncol, row_stride   slab geometry (col contiguous)
 *   skipna      mean over the non-NaN terms (NaN when there is none)
 *   out         device [nout][nrow][ncol], same element type as the inputs    */
enum { WB2_MAP_BIAS = 0, WB2_MAP_MSE = 1, WB2_MAP_MAE = 2 };
int wb2_det_maps(wb2_ctx* ctx, const void* f, const void* t, int dtype, int stat,
                 int64_t nout, int32_t ngroup, const int64_t* off_f,
                 const int64_t* off_t, int32_t nrow, int32_t ncol,
                 int64_t row_stride, int skipna, void* out);

/* Ensemble variant: SpatialCRPS / SpatialCRPSSkill / SpatialCRPSSpread
 * (metrics.py:718-772), SpatialEnsembleVariance (:1244-1266),
 * SpatialEnsembleMeanMSE / DebiasedSpatialEnsembleMeanMSE (:1366-1399) and the
 * time mean of EnsembleMetric.compute (:598-607).  One read of the members
 * yields every selected map.
 *   stat_mask   bit i selects point-wise statistic i of WB2_ENS_NSTAT's list
 *               (0 skill, 1 spread, 2 (t - xbar)^2, 3 variance, 4 debiased MSE);
 *               bit 5 = point-wise CRPS, skill - spread / 2 (metrics.py:729-739)
 *   out         device [popcount(stat_mask)][nout][nrow][ncol] float32, in
 *               increasing bit order; 1..64 members                            */
int wb2_ens_maps(wb2_ctx* ctx, const void* x, const void* t, int dtype,
                 int32_t nmember, int64_t member_stride, int64_t nout,
                 int32_t ngroup, const int64_t* off_x, const int64_t* off_t,
                 int32_t nrow, int32_t ncol, int64_t row_stride,
                 int32_t stat_mask, int skipna, float* out);

/* ---- K9: SEEPS maps ---------------------------------------------------------------
 * Replaces SpatialSEEPS.compute_chunk (metrics.py:417-513) and, for ngroup > 1,
 * the time mean of Metric.compute: dry / light / heavy categories of forecast
 * and truth precipitation, the 3 x 3 scoring matrix of the cell's
 * climatological dry fraction p1, NaN where p1 is outside (min_p1, max_p1).
 * SEEPS (the spatial mean with skipna, :516-528) is wb2_det_metrics on the maps.
 * Every operand is read in its own dtype and each comparison runs in NumPy's
 * promoted dtype: dry_threshold is rounded to f's / t's dtype, min_p1 / max_p1
 * to p1's, and the scoring matrix is formed in p1's dtype.  The maps are
 * float32(reference).
 *   f, t         device precipitation of f_dtype / t_dtype (WB2_F32 / WB2_F64)
 *   wet          device base of the climatological wet-threshold slabs, of
 *                wet_dtype;
 *   off_wet_f/t  host [nout * ngroup]: the slab for the forecast's / truth's
 *                valid time (day-of-year / hour lookup folded into the table)
 *   p1           device [nrow][ncol] mean dry fraction of p1_dtype
 *   out          device [nout][nrow][ncol] float32                               */
int wb2_seeps_maps(wb2_ctx* ctx, const void* f, int f_dtype, const void* t, int t_dtype,
                   const void* wet, int wet_dtype, const void* p1, int p1_dtype,
                   int64_t nout, int32_t ngroup,
                   const int64_t* off_f, const int64_t* off_t,
                   const int64_t* off_wet_f, const int64_t* off_wet_t,
                   int32_t nrow, int32_t ncol, int64_t row_stride,
                   int64_t wet_row_stride, double dry_threshold, double min_p1,
                   double max_p1, int skipna, float* out);

/* ---- derived variables -------------------------------------------------------------
 * wb2_wind_speed replaces WindSpeed.compute (derived_variables.py:77-99):
 * out[i] = sqrt(u[i]^2 + v[i]^2) in float32, bit-identical to NumPy; device
 * pointers, n elements.                                                          */
int wb2_wind_speed(wb2_ctx* ctx, const float* u, const float* v, float* out,
                   int64_t n);

/* wb2_wind_dynamics replaces the horizontal-derivative variables of
 * derived_variables.py:102-338 -- _d_dx / _d_dy (:102-130) and the compute() of
 * WindDivergence, WindVorticity, VerticalVelocity (:149-209) and the geostrophic
 * and ageostrophic winds (:231-338) -- one `kind` per output:            */
#define WB2_DYN_DIVERGENCE 0              /* _d_dx(u) + _d_dy(v)                    */
#define WB2_DYN_VORTICITY 1               /* _d_dx(v) - _d_dy(u)                    */
#define WB2_DYN_VERTICAL_VELOCITY 2       /* cumulative_trapezoid(-div, 100*level)  */
#define WB2_DYN_GEOSTROPHIC_WIND_SPEED 3  /* sqrt(ug^2 + vg^2)                      */
#define WB2_DYN_U_GEOSTROPHIC 4           /* ug = -_d_dy(z) / f                     */
#define WB2_DYN_V_GEOSTROPHIC 5           /* vg = _d_dx(z) / f                      */
#define WB2_DYN_AGEOSTROPHIC_WIND_SPEED 6 /* sqrt((u - ug)^2 + (v - vg)^2)          */
#define WB2_DYN_U_AGEOSTROPHIC 7          /* u - ug                                 */
#define WB2_DYN_V_AGEOSTROPHIC 8          /* v - vg                                 */
/* u, v, z   device float32 [nouter][nlev][field]; a field is nlat x nlon cells
 *           with element strides lat_stride / lon_stride, which must be
 *           (nlon, 1) -- (latitude, longitude) -- or (1, nlat) -- (longitude,
 *           latitude).  Kinds 0-2 read u and v, kinds 3-5 z, kind 6 u, v and
 *           z, kind 7 u and z, kind 8 v and z; an operand a kind does not read
 *           may be NULL.
 *   lat_coef, lon_coef  host [n][3] float64: np.gradient's coefficients per
 *           index -- index 0 and n-1: the edge spacing dx[0] / dx[n-2];
 *           interior with *_uniform != 0: 2*dx; otherwise np.gradient's a, b, c
 *           for f[i-1], f[i], f[i+1] (the spacing is uniform when every diff of
 *           the coordinate equals the first exactly, as np.gradient decides);
 *   cos_lat   host [nlat] float64 cos(deg2rad(lat));
 *   coriolis  host [nlat] float64 2 * 7.292e-5 * sin(deg2rad(lat)) (kinds 3-8);
 *   pressure  host [nlev] float64 100 * level, in storage order (kind 2);
 *   out       device float32, same shape and layout as the inputs.
 * Kinds 0, 1, 3-8 treat the nouter * nlev fields alike; kind 2 walks the nlev
 * levels of each column in one thread and integrates the float64 divergence.
 * Numerics: for float32 data on float64 coordinates every output is the
 * reference's float64 arithmetic (np.gradient with edge_order=1, no longitude
 * wrap-around; _d_dx as two float64 divisions, 0 where cos(lat) <= 1e-6;
 * _d_dy a float32 division by float32(M), M = 2 pi 6367500 / 360) rounded once
 * to float32, bit for bit, including NaN and +-inf (the geostrophic wind is
 * +-inf or NaN where f = 0).  Deviations: float64 data is cast to float32 by the
 * caller first (the reference's _d_dy would then run in float64), and float32
 * coordinates are taken as float64.  Errors: NULL operands, negative sizes, an
 * unknown kind, nlat or nlon < 2, other strides.                              */
int wb2_wind_dynamics(wb2_ctx* ctx, int kind, const float* u, const float* v,
                      const float* z, int64_t nouter, int32_t nlev, int32_t nlat,
                      int32_t nlon, int64_t lat_stride, int64_t lon_stride,
                      const double* lat_coef, int lat_uniform,
                      const double* lon_coef, int lon_uniform,
                      const double* cos_lat, const double* coriolis,
                      const double* pressure, float* out);

/* wb2_column_integral replaces the level integrals of derived_variables.py:
 * TotalColumnWater.compute (:383-385), IntegratedWaterTransport.compute (:418-430)
 * and EddyKineticEnergy.compute (:223-228), all of which end in xarray's
 * integrate('level') = sum(dx * 0.5 * (y[1:] + y[:-1]), skipna=False):      */
#define WB2_COL_TOTAL_COLUMN 0 /* (1/9.81) * S(q)                                   */
#define WB2_COL_IVT 1          /* (1/9.81) * sqrt(S(q*u)^2 + S(q*v)^2)               */
#define WB2_COL_EKE 2          /* 0.5 * S(u'^2 + v'^2), u' = u - zonal mean of u      */
/* q, u, v   device arrays of `dtype` (WB2_F32 / WB2_F64) [nouter][nlev][ninner]
 *           with outer_stride elements between outer indices (>= nlev * ninner;
 *           larger when the levels are a contiguous window of a longer axis,
 *           the pointers then start at the window's first level).  Kind 0 reads
 *           q, kind 1 q, u and v, kind 2 u and v; an operand a kind does not
 *           read may be NULL.
 *   nlon, lon_stride  kind 2 only (ignored otherwise): a level of ninner cells is
 *           nrow = ninner / nlon rows of nlon longitudes, with lon_stride 1
 *           ([nrow][nlon]) or nrow ([nlon][nrow]);
 *   weight  host [nlev - 1] float64, w_k = 0.5 * (level[k+1] - level[k]) with
 *           the level coordinate taken as float64 (may be NULL when nlev < 2);
 *   out     device [nouter][ninner] of `dtype`, the inner cells in the inputs'
 *           order.
 * Kind 2 with lon_stride 1 runs one CTA per row; with lon_stride nrow, one CTA
 * per tile of up to 8 adjacent rows, so that a warp reads adjacent rows.  Both
 * keep the level sums of their cells in shared memory: nlon * (16 + 2 *
 * sizeof(T)) bytes per CTA for lon_stride 1, tile * nlon * 16 for lon_stride
 * nrow (the tile shrinks to fit, down to 1 row).
 * Numerics, with T the data type and S(y) = sum_k w_k * f64(T(y[k] + y[k+1]))
 * accumulated in float64 from k = 0 upward, starting from the k = 0 term:
 *   kind 0  (1/9.81) * S(q), the double constant 1/9.81 times S (not S / 9.81);
 *   kind 1  y = T(q * u) and T(q * v), rounded in T as the reference's q * u;
 *           (1/9.81) * sqrt(Su^2 + Sv^2) in float64;
 *   kind 2  y_k = u'^2 + v'^2 in float64, u' = f64(u) - ubar, ubar the mean of
 *           the non-NaN cells of that level's row accumulated in float64 (NaN for
 *           an all-NaN row); the pair sum y[k] + y[k+1] is float64 too; 0.5 * S.
 * Correctly rounded operations only (no FMA contraction); the result is rounded
 * once to T.  NaN propagates through the level sum (skipna=False); nlev < 2 gives
 * 0, as trapz does.  Deviations from the reference:
 *   kinds 0 and 1  only the summation order: where `level` is the innermost axis
 *           NumPy sums the terms pairwise, so the float64 sums differ in the
 *           last bits (|dS| <= nlev * 2^-53 * sum_k |w_k p_k|); in any other layout
 *           the order is this one.  A float32 result is the reference's float64
 *           result rounded once.
 *   kind 2  the reference rounds ubar, u' and the squares to float32 and sums
 *           ubar in float32; for float32 data the gap to it is at most
 *           |dE| <= 0.5 * sum_k |w_k| (e_k + e_{k+1}), with maxima over level
 *           k's row (NaN cells left out)
 *           e_k = 2^-23 (5 max y + 2 nlon (max|u'| max|u| + max|v'| max|v|))
 *           (DESIGN.md section 8h derives it).
 * Float32 level coordinates are taken as float64.  Errors: NULL operands, negative
 * sizes, an unknown kind or dtype, outer_stride < nlev * ninner, for kind 2 an
 * ninner that is not a multiple of nlon, another lon_stride, or a row too wide for
 * shared memory.  One kernel launch per call.                                   */
int wb2_column_integral(wb2_ctx* ctx, int kind, int dtype, const void* q, const void* u,
                        const void* v, int64_t nouter, int64_t outer_stride, int32_t nlev,
                        int64_t ninner, int32_t nlon, int64_t lon_stride,
                        const double* weight, void* out);

/* wb2_lapse_rate replaces LapseRate.compute (derived_variables.py:355-362):
 *   dT_dp / dz_dp,  dT_dp = T.differentiate('level'),
 *   dz_dp = (1 / 9.81) * Z.differentiate('level').
 * t, z    device arrays of `dtype` (WB2_F32 / WB2_F64) [nouter][nlev][ninner]:
 *         temperature and geopotential in the same layout, the level axis
 *         wherever it sits (ninner = 1 when it is innermost);
 * coef    host [nlev][3] float64, np.gradient's coefficients along the level
 *         coordinate as _derived_wind.gradient_table gives them (the layout of
 *         wb2_wind_dynamics' lat_coef), `uniform` != 0 when every level step
 *         equals the first exactly;
 * out     device [nouter][nlev][ninner] of `dtype`.
 * One thread per (outer, inner) column walks its levels; consecutive threads
 * take consecutive inner cells.  With ninner < 32 (the level axis innermost)
 * one thread per cell reads its stencil instead, so a warp's loads stay
 * contiguous; the arithmetic is the same.  Numerics, with T the data type and every step
 * a correctly rounded operation (no FMA contraction):
 *   dT, dZ  np.gradient(f, level, edge_order=1) rounded once to T: the edges
 *           T(f[1] - f[0]) / dx[0] and T(f[n-1] - f[n-2]) / dx[n-2] and the
 *           uniform interior T(f[k+1] - f[k-1]) / (2 dx) as float64 divisions,
 *           the non-uniform interior (a f[k-1] + b f[k]) + c f[k+1] in float64;
 *   dz      T(1/9.81) * dZ in T (the Python scalar is weak under NEP 50);
 *   out     dT / dz in T.
 * For float32 and float64 data on an integer or float64 level coordinate this is
 * the reference's result bit for bit, NaN and +-inf included (dz == 0 gives
 * +-inf or NaN, as NumPy does).  Deviations: the caller casts integer data to
 * float64 (np.gradient does the same) and T and Z of different float types to
 * their common type (the reference would differentiate each in its own type);
 * a float32 level coordinate is taken as float64.  Errors: NULL operands,
 * negative sizes, an unknown dtype, nlev < 2.  One kernel launch per call.      */
int wb2_lapse_rate(wb2_ctx* ctx, int dtype, const void* t, const void* z, int64_t nouter,
                   int32_t nlev, int64_t ninner, const double* coef, int uniform,
                   void* out);

/* wb2_relative_humidity replaces RelativeHumidity.compute
 * (derived_variables.py:450-468), MetPy's formula with Bolton's (1980)
 * saturation vapour pressure, T in K and p in hPa:
 *   svp = 6.112 * exp(17.67 * (T - 273.15) / (T - 29.65))
 *   mr  = q / (1 - q)
 *   out = mr / (0.622 * svp / (p - svp))
 * t, q      device arrays of `dtype` (WB2_F32 / WB2_F64) [nouter][npres][ninner],
 *           temperature and specific humidity in the same layout;
 * pressure  host [npres] float64: the pressure coordinate along the npres axis
 *           (npres = 1 for a scalar coordinate), in the coordinate's own values;
 * out       device [nouter][npres][ninner] of `out_dtype`, which the caller sets
 *           to NumPy's promotion of the pressure coordinate's dtype with the
 *           data's (int64 levels and float32 data give float64, float32 levels
 *           float32); float64 data with a float32 out_dtype is rejected.
 * Long slabs (ninner >= 256) run one CTA row per (outer, p) slab, so the
 * pressure is uniform within a CTA; shorter ones a flat loop.  Numerics, with T
 * the data type and O = out_dtype, every step correctly rounded, no FMA
 * contraction, in the reference's dtypes:
 *   x    T(17.67) * (t - T(273.15)) / (t - T(29.65)) in T;
 *   e    exp(x): a float32 x is evaluated in float64 and rounded once to float32;
 *        a float64 x takes CUDA's exp, at most 1 ulp from the exact value;
 *   svp  T(6.112) * e in T;   mr = q / (T(1) - q) in T;
 *   out  O(T(0.622) * svp) / (O(p) - O(svp)), then O(mr) / that, in O.
 * NaN and +-inf propagate as in NumPy.  The gap to the reference is NumPy's own
 * exp error: its float32 exp (the AVX512F path of NumPy 2.3) lies up to 2 ulp
 * from the correctly rounded value over every float32 T in [180, 330] K, so svp
 * differs by at most 3 float32 ulp and |out - ref| <= 2^-20 |ref| (1 + |svp / (p -
 * svp)|); for float64 data both exps are within 1 ulp, and the bound is
 * 2^-49 |ref| (1 + |svp / (p - svp)|).  Deviations: the caller casts integer data
 * to float64 (NumPy's result is the same) and t and q of different float types to
 * their common type (the reference computes svp in t's type and mr in q's).
 * Errors: NULL operands, negative sizes, npres < 1, an unknown dtype or
 * out_dtype.  One kernel launch per call.                                        */
int wb2_relative_humidity(wb2_ctx* ctx, int dtype, int out_dtype, const void* t,
                          const void* q, int64_t nouter, int32_t npres, int64_t ninner,
                          const double* pressure, void* out);

/* wb2_ens_mean replaces the ensemble-mean pipeline of
 * scripts/compute_ensemble_mean.py:110-141 (xbeam.Mean(realization, skipna)):
 * out[field][cell] = mean_m x[off_x[field] + m * member_stride + cell], float32;
 * skipna: mean over the non-NaN members (NaN when there is none).  Device
 * pointers; `slab` = cells per field (contiguous); out [nfield][slab].  The mean
 * stays in HBM for K1 (ensemble-mean RMSE / ACC) -- no host round trip.        */
int wb2_ens_mean(wb2_ctx* ctx, const float* x, int32_t nmember,
                 int64_t member_stride, int64_t nfield, const int64_t* off_x,
                 int64_t slab, int skipna, float* out);

/* wb2_spectrum_interp replaces interpolate_spectral_frequencies
 * (derived_variables.py:629-682) on the output of wb2_zonal_spectrum: row `lat`
 * of a spectrum lives on the increasing frequencies freq_table[lat][k] (host
 * [nrow][nk] float64, the `frequency` coordinate of the reference's result);
 * every row is interpolated linearly to the common `freqs` (host [nfreq],
 * float64), NaN outside the row's range like xarray's .interp, with scipy
 * interp1d's interval (searchsorted side='left') and weighted form
 * ((f - x_lo) / dx) * y_hi + ((x_hi - f) / dx) * y_lo in float64: scipy's
 * value rounded to float32, NaN / inf included.
 *   spec device [nfield][nrow][nk] float32;  out device [nfield][nrow][nfreq]    */
int wb2_spectrum_interp(wb2_ctx* ctx, const float* spec, int64_t nfield,
                        int32_t nrow, int32_t nk, const double* freq_table,
                        int32_t nfreq, const double* freqs, float* out);

/* ---- day-of-year climatology --------------------------------------------------------
 * wb2_climatology replaces compute_hourly_stat / compute_daily_stat (the
 * `explicit` method, weatherbench2/utils.py:88-166) and compute_hourly_stat_fast
 * / compute_daily_stat_fast (`fast`, utils.py:169-287) for the statistics mean
 * and std of scripts/compute_climatology.py.  The series x is [time][ncell]
 * (cells contiguous, float32 or float64); the host describes the selection:
 *   nres > 0   x is first resampled to days: day i = skip-NaN mean of the
 *              res_count[i] consecutive slabs from res_start[i] (host, NaN when
 *              the count is 0; float32 input only), and the tables below index
 *              those days instead of x's time steps
 *   items      host [nhour][nday][nitem]: the steps feeding day slot d of hour h
 *              (explicit: the value of stacked year j; fast: any step with that
 *              day-of-year label), -1 = missing
 *   fill       host [nhour][nitem]: the day-365 step of stacked year j (-1 =
 *              none) that replaces a NaN / missing item (explicit only, else
 *              ignored; utils.py:105)
 *   hour_nday  host [nhour]: day slots of hour h, the period of the circular
 *              window (the window wraps positionally over slots 0..n-1)
 *   out_row    host [nhour][nday]: output row of each slot, < nday_out, distinct
 *              within an hour (a repeated row is an error); rows an hour does
 *              not produce are NaN
 *   method     0 explicit: xarray's weighted mean / population std over (window,
 *              year) with the triangular weights of create_window_weights
 *              1 fast: per-slot mean / std (ddof 0), then the mean over the
 *              window of weight * value, NaN skipped (count denominator)
 *   mean, std  device [nhour][nday_out][ncell] float32; either may be NULL
 * Moments accumulate in float64 around a per-cell shift (a finite value of the
 * cell among up to 512 table entries spread over the hour's table, the fill
 * applied); one read of x serves both statistics.  window_size: odd, >= 3.      */
int wb2_climatology(wb2_ctx* ctx, const void* x, int dtype, int64_t ntime,
                    int64_t ncell, int64_t nres, const int64_t* res_start,
                    const int32_t* res_count, int32_t nhour, int32_t nday,
                    int32_t nitem, const int64_t* items, const int64_t* fill,
                    const int32_t* hour_nday, const int32_t* out_row,
                    int32_t nday_out, int32_t window_size, int32_t method,
                    float* mean, float* std);

/* wb2_climatology on a HOST series (NumPy / memmap): bands of cells, each band's
 * selected time rows in one strided 2-D copy, double buffered so that the copy
 * of band b+1 overlaps the kernels of band b.  `budget` bounds the device bytes
 * of the two staging buffers (at least one cell per band).  mean / std are host
 * [nhour][nday_out][ncell] float32.                                              */
int wb2_climatology_host(wb2_ctx* ctx, const void* x, int dtype, int64_t ntime,
                         int64_t ncell, int64_t nres, const int64_t* res_start,
                         const int32_t* res_count, int32_t nhour, int32_t nday,
                         int32_t nitem, const int64_t* items, const int64_t* fill,
                         const int32_t* hour_nday, const int32_t* out_row,
                         int32_t nday_out, int32_t window_size, int32_t method,
                         size_t budget, float* mean, float* std);

/* wb2_climatology_quantile replaces Quantile.compute and SEEPSThreshold.compute
 * (scripts/compute_climatology.py:130-177) passed as stat_fn to
 * compute_hourly_stat / compute_daily_stat (weatherbench2/utils.py:88-166), the
 * `explicit` method only.  The series and the tables are those of
 * wb2_climatology (method 0, `fill` required).  Per output value the samples are
 * the nyear x window_size entries of the wrapped window, the day-365 fill
 * applied, tap j weighted by create_window_weights (utils.py:73-85), and the
 * statistic is xarray's weighted type-7 quantile over (window, year): NaN and
 * zero-weight samples dropped, nw = (sum w)^2 / sum w^2, c = [0, cumsum(w/sum w)]
 * over the sorted values, h = clip((nw-1) q + 1, 1, nw),
 * v = max((h-1)/nw, min(h/nw, c)) nw - h + 1, result sum_i x_i (v[i+1] - v[i]),
 * NaN without samples.
 *   quantiles  host [nquantile] in [0, 1], 1 <= nquantile <= 16
 *   seeps      0: out = the quantiles, dry_fraction must be NULL
 *              1: samples x < dry_threshold (compared in the series' precision)
 *                 are dropped like NaN before the quantiles, and dry_fraction =
 *                 the unweighted mean of (x < dry_threshold) over all
 *                 nyear * window_size samples (NaN is not dry; nyear of hour h
 *                 = the item columns with a step in some slot of the hour, so
 *                 an hour without any is NaN); SEEPSThreshold is nquantile 1,
 *                 quantiles {2/3}
 *   out        device [nhour][nquantile][nday_out][ncell] float32
 *   dry_fraction  device [nhour][nday_out][ncell] float32 (seeps 1)
 * nitem * window_size <= 8192.                                                   */
int wb2_climatology_quantile(wb2_ctx* ctx, const void* x, int dtype, int64_t ntime,
                             int64_t ncell, int64_t nres, const int64_t* res_start,
                             const int32_t* res_count, int32_t nhour, int32_t nday,
                             int32_t nitem, const int64_t* items, const int64_t* fill,
                             const int32_t* hour_nday, const int32_t* out_row,
                             int32_t nday_out, int32_t window_size, int32_t nquantile,
                             const double* quantiles, int32_t seeps, double dry_threshold,
                             float* out, float* dry_fraction);

/* wb2_climatology_quantile on a HOST series, streamed in bands of cells like
 * wb2_climatology_host; out / dry_fraction are host arrays of the same layout. */
int wb2_climatology_quantile_host(wb2_ctx* ctx, const void* x, int dtype, int64_t ntime,
                                  int64_t ncell, int64_t nres, const int64_t* res_start,
                                  const int32_t* res_count, int32_t nhour, int32_t nday,
                                  int32_t nitem, const int64_t* items, const int64_t* fill,
                                  const int32_t* hour_nday, const int32_t* out_row,
                                  int32_t nday_out, int32_t window_size, int32_t nquantile,
                                  const double* quantiles, int32_t seeps,
                                  double dry_threshold, size_t budget, float* out,
                                  float* dry_fraction);

/* ---- time resampling and rolling windows ------------------------------------------
 * wb2_time_window_stats replaces xarray's resample(...).mean/min/max/sum and
 * rolling(..., min_periods=None).mean/min/max/sum along one axis, the computation
 * of scripts/resample_in_time.py.  x is [nouter][ntime][ninner] (float32 or
 * float64, read in place: a forecast resampled along prediction_timedelta has
 * outer = time, inner = the cells after it).  Exactly one of:
 *   bins      resample: bin_start / bin_count host [nbin]; output b reduces the
 *             bin_count[b] steps from bin_start[b].  Bins are in order and
 *             disjoint (bin_start[b] >= bin_start[b-1] + bin_count[b-1]),
 *             bin_count >= 0, and lie inside [0, ntime) (an empty bin's start is
 *             at most ntime).  window must be 0.
 *   window    rolling, > 0: output t reduces steps [t - window + 1, t]; nbin must
 *             be 0 and the bin arrays NULL.  There are ntime outputs.
 * Per output (mean / min / max / sum):
 *   resample, skipna 0   any NaN in the bin -> NaN
 *   resample, skipna 1   NaN skipped; an all-NaN bin gives NaN, except sum = 0
 *   empty bin            NaN for every statistic, sum included
 *   rolling              NaN when t < window - 1 or when any value of the window is
 *                        NaN, whatever skipna is (window > ntime: all NaN)
 *   +-Inf                as NumPy float64 over the window: mean([1, inf]) = inf,
 *                        inf + -inf = nan; a window that slid past an Inf is finite
 * Mean and sum accumulate in float64; min and max are one of the window's values.
 *   mean, min, max, sum  device [nouter][nout][ninner] of x's dtype (nout = nbin,
 *                        or ntime for rolling); NULL = not wanted, at least one
 *                        given                                                       */
int wb2_time_window_stats(wb2_ctx* ctx, const void* x, int dtype, int64_t nouter,
                          int64_t ntime, int64_t ninner, int64_t nbin,
                          const int64_t* bin_start, const int32_t* bin_count,
                          int32_t window, int skipna, void* mean, void* min, void* max,
                          void* sum);

/* wb2_time_window_stats on a HOST series (NumPy / memmap): bands of inner cells of
 * one outer index (or of whole outer indices when they fit), each band in one
 * strided 2-D copy, double buffered so that the copy of band b+1 overlaps the
 * kernel of band b; every output band is copied back.  `budget` bounds the device
 * bytes of the two staging buffers (at least one cell per band).  mean / min /
 * max / sum are host arrays of the same layout.                                    */
int wb2_time_window_stats_host(wb2_ctx* ctx, const void* x, int dtype, int64_t nouter,
                               int64_t ntime, int64_t ninner, int64_t nbin,
                               const int64_t* bin_start, const int32_t* bin_count,
                               int32_t window, int skipna, size_t budget, void* mean,
                               void* min, void* max, void* sum);

/* ---- precipitation accumulations over lead time -----------------------------------
 * wb2_precip_accumulation replaces PrecipitationAccumulation.compute
 * (weatherbench2/derived_variables.py:471-528): diff along the lead axis, a rolling
 * sum of `window` differences, negative sums set to 0, a NaN step in front.  x is a
 * cumulative series [nouter][ntime][ninner] (float32 or float64, read in place, so
 * any C-contiguous array with the lead axis in the middle); out is device
 * [nouter][ntime][ninner] of x's dtype T.  Per output step t:
 *   t < window      NaN (every output is NaN when window >= ntime)
 *   otherwise       d[k] = T(x[k] - x[k-1]), rounded in T as xarray's diff does;
 *                   s = d[t-w+1] + d[t-w+2] + ... + d[t] accumulated in float64 in
 *                   that order (oldest first), rounded once to T
 *   clamp_negative  a rounded sum < 0 becomes +0.0; NaN stays NaN and -0.0 is kept
 * NaN and +-Inf follow from that arithmetic: a NaN anywhere in x[t-w .. t] gives
 * NaN, an Inf inside the window gives inf + -inf = NaN.  The reference sums float32
 * data in float32; the gap to it is at most (w + 1) 2^-24 sum |d[k]|.  window must
 * be >= 1 and at most 1024 unless window >= ntime.  One kernel launch per call.   */
int wb2_precip_accumulation(wb2_ctx* ctx, const void* x, int dtype, int64_t nouter,
                            int64_t ntime, int64_t ninner, int32_t window,
                            int clamp_negative, void* out);

/* wb2_precip_accumulation on a HOST series (NumPy / memmap), streamed in bands like
 * wb2_time_window_stats_host within `budget` device bytes; out is a host array of
 * the same layout.                                                                  */
int wb2_precip_accumulation_host(wb2_ctx* ctx, const void* x, int dtype, int64_t nouter,
                                 int64_t ntime, int64_t ninner, int32_t window,
                                 int clamp_negative, size_t budget, void* out);

/* ---- quantiles over a sample axis ---------------------------------------------------
 * wb2_quantile replaces xarray's Dataset.quantile(q, dim, skipna) (method 'linear'),
 * the computation of scripts/compute_quantiles.py:168-183.  x is
 * [nouter][nsample][ninner] (float32 or float64, read in place); quantiles is a HOST
 * array of nquantile float64 values in [0, 1]; out is device
 * [nquantile][nouter][ninner] float64.  Per cell, with T the data type, the result is
 * numpy's np.quantile (skipna 0) / np.nanquantile (skipna 1) with float64 q, bit for
 * bit:
 *   1. skipna 0 and any sample NaN: every output NaN.  skipna 1: NaN samples are
 *      dropped.  m = the samples left; m = 0 gives NaN for every output.
 *   2. s = the m samples sorted ascending (equal values in any order).
 *   3. v = double(m - 1) * q, correctly rounded.  v >= m - 1: i = j = m - 1 and
 *      g = v + 1 (numpy's previous index -1).  Otherwise i = floor(v), j = i + 1,
 *      g = v - i.
 *   4. d = T(s[j] - s[i]), rounded in T.
 *   5. g < 0.5: out = double(s[i]) + double(d) * g; else
 *      out = double(s[j]) - double(d) * (1 - g); each operation a separately rounded
 *      double operation, none contracted.
 *   6. out is float64 for both data types.
 * So [inf] gives NaN, [1, inf] NaN at q = 0 and q = 1, and float32 [1, 16777218]
 * gives 8388610 at q = 0.5.  Only the sign of a zero read from samples whose +-0
 * order is undefined may differ from numpy.  Argument errors (each names the
 * argument; nothing is launched): dtype, nsample < 1, nquantile outside 1..128, a
 * quantile outside [0, 1] or NaN, a NULL pointer.  nsample and the ranks are 64-bit;
 * nouter * ninner = 0 is a no-op.  One kernel launch per call.                      */
int wb2_quantile(wb2_ctx* ctx, const void* x, int dtype, int64_t nouter, int64_t nsample,
                 int64_t ninner, int32_t nquantile, const double* quantiles, int skipna,
                 double* out);

/* wb2_quantile on a HOST series (NumPy / memmap), streamed in bands like
 * wb2_time_window_stats_host within `budget` device bytes; out is a host array of
 * the same [nquantile][nouter][ninner] layout.  One launch per band.               */
int wb2_quantile_host(wb2_ctx* ctx, const void* x, int dtype, int64_t nouter,
                      int64_t nsample, int64_t ninner, int32_t nquantile,
                      const double* quantiles, int skipna, size_t budget, double* out);

/* ---- means and raw moments over reduced dims ----------------------------------------
 * wb2_average replaces the `v * weights` + xbeam.Mean(dims, skipna) of
 * scripts/compute_averages.py and the means of compute_statistical_moments.py's
 * moment_reduce.  x (float32 or float64 T, read in place) is [k0][r0][k1][r1][k2]: the
 * k extents are kept, the r extents reduced (any extent may be 1).  Per kept cell
 * (k0, k1, k2), with n = r0 * r1 samples x[s] in the flat order s = r0' * r1 + r1':
 *   w[s]     weights == NULL: 1; else the HOST float64 table weights[(s / wdiv) % wlen]
 *            (wdiv * wlen must divide n)
 *   y[s]     double(x[s]) * w[s], one float64 multiply
 *   z[s]     double(T(x[s] * x[s])) * w[s]: the square is rounded in T as np.square
 *            does (a float32 square may overflow to inf)
 *   skipna 1 a NaN x[s] contributes +0.0 to both sums; skipna 0 it propagates
 *   N        the number of non-NaN x[s]; count = N (skipna 1) or n (skipna 0)
 *   mean     = S1 / count, mean_sq = S2 / count, frac = N / n (float64 divisions)
 * The divisor is the count, not sum w: the reference's `v * weights` + xbeam.Mean.
 * A cell with count 0 gives NaN; Inf follows IEEE float64 (inf + -inf is NaN).
 * S1 (S2 likewise) is summed in float64 in this order, fixed by n alone:
 *   1. the samples are cut into chunks of 65536 consecutive s;
 *   2. in a chunk, class c (0..31) adds y[s] for s = chunk start + c, + 32, ... in
 *      increasing s to an accumulator starting at +0.0;
 *   3. the 32 class sums are added pairwise: a[c] + a[c + 16] for c < 16, then the
 *      same with 8, 4, 2, 1 (a xor butterfly), giving the chunk's partial;
 *   4. the partials are added in chunk order starting from +0.0.
 * No addition chain is longer than ceil(n / 32) + 7, so the sum is within
 * (ceil(n / 32) + 7) 2^-53 sum |y[s]| of the exact sum of the y[s] (to first order).
 * Outputs (device arrays [k0][k1][k2]; each may be NULL, not all three): mean and
 * mean_sq are float64 when weighted, else T, each rounded once from the float64
 * quotient; frac is float64.  Argument errors (each names the argument; nothing is
 * launched): dtype, r0 or r1 < 1, a negative kept extent, weights that do not fit
 * the sample index, no output requested, a NULL pointer.  k0 * k1 * k2 = 0 is a
 * no-op.  One kernel launch per call when n <= 65536, else three.                 */
int wb2_average(wb2_ctx* ctx, const void* x, int dtype, int64_t k0, int64_t r0, int64_t k1,
                int64_t r1, int64_t k2, const double* weights, int64_t wdiv, int64_t wlen,
                int skipna, void* mean, void* mean_sq, double* frac);

/* wb2_average on a HOST array (NumPy / memmap), streamed through two staging buffers
 * within `budget` device bytes.  Bands hold whole cells: whole k0 slabs, else k1
 * slices [r0][m][r1][k2] of one k0, else k2 cells [r0][r1][nb] of one (k0, k1); the
 * outputs are host arrays of the same layout, bit-equal to wb2_average's.  Only a
 * budget below one cell (its r0 * r1 samples, outputs and chunk partials, twice) is
 * an error naming it.  The device entry's launches per band.                       */
int wb2_average_host(wb2_ctx* ctx, const void* x, int dtype, int64_t k0, int64_t r0,
                     int64_t k1, int64_t r1, int64_t k2, const double* weights, int64_t wdiv,
                     int64_t wlen, int skipna, size_t budget, void* mean, void* mean_sq,
                     double* frac);

/* ---- K10: rank histogram ---------------------------------------------------------
 * Replaces RankHistogram.compute_chunk (metrics.py:1894-2042) and the time mean
 * of EnsembleMetric.compute: rank of the truth among the members (NaN last),
 * binned into nbins (nbins divides nmember + 1), one-hot per grid point or,
 * for ngroup > 1, the mean of the one-hots over the group.  random_ties != 0
 * places the truth uniformly among members exactly equal to it (the effect of
 * the reference's tie-breaking noise) using a counter-based hash of `seed`.
 *   out   device [nout][nrow][ncol][nbins] float32                                */
int wb2_rank_histogram(wb2_ctx* ctx, const float* x, const float* t,
                       int32_t nmember, int64_t member_stride, int64_t nout,
                       int32_t ngroup, const int64_t* off_x, const int64_t* off_t,
                       int32_t nrow, int32_t ncol, int64_t row_stride,
                       int32_t nbins, int32_t random_ties, uint64_t seed,
                       float* out);

/* ---- K7: threshold ("binary event") and Gaussian-forecast metrics -------------
 * wb2_ens_threshold_metrics replaces EnsembleBrierScore /
 * DebiasedEnsembleBrierScore (metrics.py:1523-1710), EnsembleIgnoranceScore
 * (:1713-1790) and EnsembleRPS (:1793-1891) .compute_chunk: one read of the
 * members yields all four point-wise scores for every threshold.
 * Thresholds, two forms:
 *   thr_b == NULL  thr_a is a float32 threshold field per (threshold, field):
 *                  off_a host [nthreshold][nfield]  (QuantileThreshold,
 *                  thresholds.py:118-149)
 *   thr_b != NULL  thr_a / thr_b are the climatological mean / std slabs,
 *                  off_a / off_b host [nfield], z host [nthreshold] =
 *                  norm.ppf(quantile): thr = mean + z * std in float64
 *                  (GaussianQuantileThreshold, thresholds.py:152-185)
 *   out   device [nfield][nthreshold][nregion][8] float64:
 *         [0] sum W*brier  [1] sum W*debiased brier  [2] sum W*ignorance
 *         [3] sum W*rps part   [4..7] the matching weight sums
 * Any number of members (streamed, not held in registers).                      */
int wb2_ens_threshold_metrics(wb2_ctx* ctx, const void* x, const void* t,
                              int dtype, int32_t nmember, int64_t member_stride,
                              int64_t nfield, const int64_t* off_x,
                              const int64_t* off_t, int32_t nthreshold,
                              const void* thr_a, const int64_t* off_a,
                              const void* thr_b, const int64_t* off_b,
                              const double* z, const wb2_weights* w, int skipna,
                              double* out);

/* Map-output variant: SpatialEnsembleBrierScore (metrics.py:1615-1637),
 * SpatialDebiasedEnsembleBrierScore (:1701-1710), SpatialEnsembleIgnoranceScore
 * (:1768-1790), SpatialEnsembleRPS (:1868-1891) and the time mean of
 * EnsembleMetric.compute (:598-607): fields grouped like wb2_det_maps
 * (off_* host [nout * ngroup], field thresholds [nthreshold][nout * ngroup]).
 *   stat  0 brier | 1 debiased brier | 2 ignorance | 3 rps part
 *   out   device [nthreshold][nout][nrow][ncol] float32                          */
int wb2_ens_threshold_maps(wb2_ctx* ctx, const void* x, const void* t, int dtype,
                           int32_t nmember, int64_t member_stride, int64_t nout,
                           int32_t ngroup, const int64_t* off_x,
                           const int64_t* off_t, int32_t nthreshold,
                           const void* thr_a, const int64_t* off_a,
                           const void* thr_b, const int64_t* off_b,
                           const double* z, int32_t nrow, int32_t ncol,
                           int64_t row_stride, int32_t stat, int skipna,
                           float* out);

/* wb2_gaussian_metrics replaces GaussianCRPS / GaussianVariance
 * (metrics.py:849-937) when nthreshold == 0:
 *         out [nfield][1][nregion][8]: [0] sum W*crps [1] sum W*std^2, [4],[5] weights
 * and GaussianBrierScore / GaussianIgnoranceScore / GaussianRPS (:963-1158)
 * when nthreshold > 0 (thresholds as above):
 *         out [nfield][nthreshold][nregion][8]: [0] brier [2] ignorance [3] rps part
 * Point-wise math: the reference calls scipy.stats.norm in float64; here z is
 * rounded to float32 and erfcf / expf / logf / log1pf run in float32 (a few ulp
 * relative on min(cdf, 1 - cdf)); where that tail is below 1e-7 (|z| > 5.2) it
 * is recomputed in float64 from the float32 z and the reference's float64
 * `1 - cdf` is replayed, so the ignorance is inf where the reference's is
 * (tail <= 2^-54) except in a band of about z^2 * 2^-22 relative around it. */
int wb2_gaussian_metrics(wb2_ctx* ctx, const void* mean, const void* std,
                         const void* t, int dtype, int64_t nfield,
                         const int64_t* off_mean, const int64_t* off_std,
                         const int64_t* off_t, int32_t nthreshold,
                         const void* thr_a, const int64_t* off_a,
                         const void* thr_b, const int64_t* off_b,
                         const double* z, const wb2_weights* w, int skipna,
                         double* out);

/* ---- K5: conservative regridding -------------------------------------------
 * Replaces ConservativeRegridder.regrid_array (= _nanmean,
 * weatherbench2/regridding.py:502-536).  The two weight matrices
 * (regridding.py:341-373, 462-499) are banded; they are passed in CSR form
 * built by the Python operator with the reference's own formulas.
 * Input slabs are (lon_src, lat_src) with lat contiguous, output slabs
 * (lon_tgt, lat_tgt) float32, exactly the reference's layout (regridding.py:190).
 * A NaN weight row (target cell not covered, regridding.py:367-371) is flagged
 * by nan_row and yields NaN; a row without taps that is not flagged gives
 * 0 / 0 = NaN.
 * Banded semantics: a target cell sees only its own stored taps, NaN inputs
 * are missing, and +-inf propagate in IEEE arithmetic (+inf and -inf in one
 * footprint give NaN).  The reference contracts with the dense matrices, where
 * 0 * inf turns the whole 2-D slice NaN; here only the cells whose footprint
 * holds the infinity are affected, whichever kernel runs.
 */
typedef struct {
  int32_t n_src;            /* source axis length                              */
  int32_t n_tgt;            /* target axis length                              */
  const int32_t* row_ptr;   /* host [n_tgt + 1] CSR offsets, row_ptr[0] = 0,
                               non-decreasing; uncovered rows have zero taps
                               and nan_row[i] = 1                              */
  const int32_t* col_idx;   /* host [nnz] source indices, strictly increasing
                               within each row (rejected otherwise)            */
  const float* val;         /* host [nnz] weights (rows sum to 1)              */
  const uint8_t* nan_row;   /* host [n_tgt] 1 = output NaN                     */
} wb2_csr;

int wb2_regrid_conservative(wb2_ctx* ctx, const float* src, float* dst,
                            int64_t nfield, int64_t src_field_stride,
                            int64_t dst_field_stride, const wb2_csr* lon_w,
                            const wb2_csr* lat_w);

/* wb2_regrid_conservative on host buffers: groups of fields in, regridded
 * groups out (H2D, kernel and D2H of neighbouring groups overlap).             */
int wb2_regrid_conservative_host(wb2_ctx* ctx, const float* src, float* dst,
                                 int64_t nfield, int64_t src_field_stride,
                                 int64_t dst_field_stride, const wb2_csr* lon_w,
                                 const wb2_csr* lat_w);

/* ---- K8: nearest-neighbour and bilinear regridding -----------------------------
 * wb2_regrid_gather replaces NearestRegridder.regrid_array
 * (regridding.py:231-247): dst[k] = src[indices[k]], `indices` host [ntarget]
 * into the raveled (lon, lat) source slab (BallTree / haversine nearest
 * neighbours, computed by the binder like regridding.py:212-228).
 * wb2_regrid_bilinear replaces BilinearRegridder.regrid_array (:256-294): per
 * target longitude a / latitude c two source taps i0, i1 and the fraction
 * t = delta / dx of jnp.interp (host arrays): i0 = -1 is NaN (outside the
 * source; i1 must then be -1 too); t < 0 returns fp[i0] untouched (jnp.interp's
 * `where` at clamped ends and at |dx| <= spacing(eps); the binder passes
 * i1 = i0, t = -1); otherwise fp[i0] + t * (fp[i1] - fp[i0]) with three
 * separate float32 roundings.  Latitude is interpolated first, then longitude;
 * taps outside [-1, n), or with only one of i0 / i1 at -1, are rejected.
 * Slabs are (lon, lat) with lat contiguous; strides in elements.               */
int wb2_regrid_gather(wb2_ctx* ctx, const float* src, float* dst, int64_t nfield,
                      int64_t src_field_stride, int64_t dst_field_stride,
                      int32_t nsource, int32_t ntarget, const int32_t* indices);
int wb2_regrid_bilinear(wb2_ctx* ctx, const float* src, float* dst,
                        int64_t nfield, int64_t src_field_stride,
                        int64_t dst_field_stride, int32_t nlon_s, int32_t nlat_s,
                        int32_t nlon_t, int32_t nlat_t, const int32_t* lon_i0,
                        const int32_t* lon_i1, const float* lon_t,
                        const int32_t* lat_i0, const int32_t* lat_i1,
                        const float* lat_t);

/* ---- K4: zonal energy spectrum ---------------------------------------------
 * Replaces ZonalEnergySpectrum.compute (weatherbench2/derived_variables.py:
 * 592-626): rfft(norm='forward') along longitude, |F_k|^2 * (1 if k==0 else 2),
 * times `scale[row]` (the latitude circumference, derived_variables.py:626).
 *   x      device [nfield][nrow][ncol] float32, ncol = number of longitudes
 *   scale  host [nrow] float64
 *   out    device float32; accumulate == 0: [nfield][nrow][ncol/2+1] written;
 *          accumulate == 1: out has [nfield_out][nrow][ncol/2+1] and field i
 *          is ADDED to slot  i % nfield_out  (device-side time-sum for the
 *          script's `xbeam.Mean(['time'])`,
 *          scripts/compute_zonal_energy_spectrum.py:234)
 * Each row is transformed as x - x[0] (x[0] added back to bin 0), so the
 * float32 rounding scales with the row's variation, not its mean.  Per bin,
 * with u = 2^-24, D = max|x_n - mean|, F_k the exact DFT of the float32 row:
 *   |got_k - want_k| <= c_k scale (2 |F_k| e + e^2) + m u want_k,
 *   e = C_plan u D,  C_plan = 2 L / sqrt(N / 2)  (DESIGN.md K4: L, m, bin 0).
 */
int wb2_zonal_spectrum(wb2_ctx* ctx, const float* x, int64_t nfield,
                       int32_t nrow, int32_t ncol, const double* scale,
                       float* out, int32_t accumulate, int64_t nfield_out);

/* K4 with the weighted meridional reduction fused in (BASELINE north star: "a
 * shared-memory rFFT along longitude followed by a weighted meridional
 * reduction").  The reference keeps `latitude` (derived_variables.py:592-626);
 * its callers average the per-latitude spectra over latitude bands afterwards,
 * so the reduction is defined on the reference's own output:
 *     out[slot][k] = sum_{fields i of the slot} sum_row scale[row] * S_ref[i][row][k]
 * where S_ref is the spectrum WITHOUT the circumference factor, i.e. the caller
 * passes scale[row] = circumference(row) * w(row) with w the (normalised)
 * latitude weight of weatherbench2/metrics.py:40-60 (or a latitude-band mask
 * times it; rows whose scale is 0 are skipped, so NaN / inf outside a band
 * do not reach it).  Fields are slot-minor like wb2_zonal_spectrum's accumulate mode
 * (field i belongs to slot i % nfield_out), so a time mean is the same call.
 *   out    device [nfield_out][ncol/2+1] float32, overwritten
 * The per-latitude spectrum is never written: 4 B read per cell, ~0 written. */
int wb2_zonal_spectrum_latsum(wb2_ctx* ctx, const float* x, int64_t nfield,
                              int32_t nrow, int32_t ncol, const double* scale,
                              float* out, int64_t nfield_out);

/* wb2_zonal_spectrum / wb2_zonal_spectrum_latsum on host buffers.  x host
 * [nfield][nrow][ncol] dense; out host, OVERWRITTEN: accumulate == 0:
 * [nfield][nrow][ncol/2+1]; accumulate != 0: the sum over the fields of each
 * slot, [nfield_out][nrow][ncol/2+1] (the accumulator stays in HBM, only the
 * sum comes back); latsum: [nfield_out][ncol/2+1].                             */
int wb2_zonal_spectrum_host(wb2_ctx* ctx, const float* x, int64_t nfield,
                            int32_t nrow, int32_t ncol, const double* scale,
                            float* out_host, int32_t accumulate,
                            int64_t nfield_out);
int wb2_zonal_spectrum_latsum_host(wb2_ctx* ctx, const float* x, int64_t nfield,
                                   int32_t nrow, int32_t ncol,
                                   const double* scale, float* out_host,
                                   int64_t nfield_out);

/* ---- slab gather: reindexing in time --------------------------------------------
 * wb2_slab_gather is the copy of weatherbench2_b200/reindexing.py (the
 * reference's expand_climatology.py, index_on_valid_time.py and
 * compute_probabilistic_climatological_forecasts.py):
 *   out[s][i] = offsets[s] < 0 ? NaN : (out_dtype) src[offsets[s] + i],
 *   0 <= s < nslab, 0 <= i < slab
 * src        device array of src_dtype (WB2_F32 / WB2_F64) of src_elems elements
 * offsets    host [nslab]; a negative entry fills its slab with NaN, any other
 *            must satisfy offsets[s] + slab <= src_elems.  The whole table is
 *            checked before anything is launched.
 * out        device [nslab][slab] of out_dtype (WB2_F32 / WB2_F64); float64 to
 *            float32 rounds to nearest (NumPy's astype), so the result is exact.
 * slab == 0 or nslab == 0 launches nothing.  Slabs of 4096 elements or more are
 * copied by CTAs of 4096 elements with 16-byte accesses where source and output
 * alignment allow; shorter slabs by CTAs over the flattened output.            */
int wb2_slab_gather(wb2_ctx* ctx, const void* src, int src_dtype, int64_t src_elems,
                    int64_t slab, int64_t nslab, const int64_t* offsets, void* out,
                    int out_dtype);

/* wb2_slab_gather on a HOST source (NumPy / memmap) into a HOST out, in bands of
 * consecutive output slabs, double buffered.  Each band uploads every distinct
 * source range it references once (ranges that touch or overlap are one copy),
 * so a source slab no output references is never read; a slab that does not fit
 * is split into pieces.  `budget` bounds the device bytes of the two staging
 * buffers; it must hold at least one element in each.                          */
int wb2_slab_gather_host(wb2_ctx* ctx, const void* src, int src_dtype, int64_t src_elems,
                         int64_t slab, int64_t nslab, const int64_t* offsets, size_t budget,
                         void* out, int out_dtype);

#ifdef __cplusplus
}
#endif
#endif /* WB2B200_H_ */

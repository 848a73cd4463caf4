"""CPU oracle for the WeatherBench2 hot path -- TEST INFRASTRUCTURE ONLY.

This module is a NumPy restatement of the reference algorithms named in
SURVEY.md section 8 (metrics / regions / conservative regridder / zonal energy
spectrum).  It is the *checker*: only ``tests/``, ``__graft_entry__.smoke()``
and ``bench.py``'s ``cpu_baseline`` / ``--impl reference`` legs may import it.
The product package (``weatherbench2_b200``) never imports anything from
``oracle/``; its numerical path is the CUDA library behind the C ABI in
``include/wb2b200.h`` and it fails loudly when that library is missing.

Parity status: **pinned** (1) against every known-answer value the reference's
own tests hold for this path (``tests/test_oracle_golden.py`` lists them with
the reference test file:line) and (2) against vectors produced by EXECUTING the
reference's own modules
(``tests/golden/make_reference_vectors.py`` -> ``reference_run_vectors.npz``,
checked by ``tests/test_reference_run_vectors.py``): metrics.py, regions.py,
thresholds.py, derived_variables.py, regridding.py and evaluation.py, imported
from a checkout of the reference and run on stand-ins for the libraries it
needs (xarray -> a re-implemented subset, jax.numpy -> NumPy with
32-bit results, apache_beam / xarray_beam -> import stubs).  Those vectors pin
the REFERENCE logic restated here; what xarray (>=2024.11), NumPy (>=2.1) and
JAX do underneath the reference's calls remains restated, operation for
operation, both in that stand-in and -- independently -- in this module.  Each function cites the reference lines it follows
(paths relative to the reference checkout).

Everything works on plain ``numpy`` arrays plus a tuple of dimension names
(``dims``), i.e. the information an ``xarray.DataArray`` carries.
"""

from __future__ import annotations

import dataclasses
from typing import Optional, Sequence, Union

import numpy as np

EARTH_RADIUS_M = 1000 * (6357 + 6378) / 2  # weatherbench2/schema.py:59

LAT = "latitude"
LON = "longitude"


# ----------------------------------------------------------------------------
# Latitude weights -- weatherbench2/metrics.py:35-60
# ----------------------------------------------------------------------------
def _assert_increasing(x: np.ndarray):
  # metrics.py:35-37
  if not (np.diff(x) > 0).all():
    raise ValueError(f"array is not increasing: {x}")


def _latitude_cell_bounds(x: np.ndarray) -> np.ndarray:
  # metrics.py:40-42 (radians; keeps x.dtype)
  pi_over_2 = np.array([np.pi / 2], dtype=x.dtype)
  return np.concatenate([-pi_over_2, (x[:-1] + x[1:]) / 2, pi_over_2])


def _cell_area_from_latitude(points: np.ndarray) -> np.ndarray:
  # metrics.py:45-52
  bounds = _latitude_cell_bounds(points)
  _assert_increasing(bounds)
  upper = bounds[1:]
  lower = bounds[:-1]
  return np.sin(upper) - np.sin(lower)


def get_lat_weights(latitude: np.ndarray) -> np.ndarray:
  """metrics.py:55-60.  `latitude` in degrees, strictly increasing."""
  weights = _cell_area_from_latitude(np.deg2rad(np.asarray(latitude)))
  weights = weights / np.mean(weights)
  return weights


# ----------------------------------------------------------------------------
# Regions -- weatherbench2/regions.py:40-158
# ----------------------------------------------------------------------------
def _label_slice_indices(coord: np.ndarray, s: slice) -> np.ndarray:
  """Indices selected by ``.sel(dim=slice(lo, hi))`` on a monotonic increasing
  float index (pandas `Index.slice_indexer`: both ends inclusive; labels need
  not be present).  regions.py:79-84 rely on this rule."""
  coord = np.asarray(coord)
  if s.step is not None:
    raise ValueError("slice steps are not used by the reference")
  start = 0 if s.start is None else int(np.searchsorted(coord, s.start, "left"))
  stop = (
      coord.size if s.stop is None
      else int(np.searchsorted(coord, s.stop, "right"))
  )
  return np.arange(start, max(start, stop))


@dataclasses.dataclass
class SliceRegion:
  """regions.py:57-95."""
  lat_slice: Union[slice, list] = dataclasses.field(
      default_factory=lambda: slice(None, None))
  lon_slice: Union[slice, list] = dataclasses.field(
      default_factory=lambda: slice(None, None))


@dataclasses.dataclass
class ExtraTropicalRegion:
  """regions.py:98-109 (note the hard-coded 20 at :108)."""
  threshold_lat: Optional[float] = 20


@dataclasses.dataclass
class LandRegion:
  """regions.py:112-138.  `land_sea_mask` has dims (latitude, longitude);
  `latitude` / `longitude` are its coordinate labels (needed only when the
  region follows a SliceRegion inside a CombinedRegion)."""
  land_sea_mask: np.ndarray
  threshold: Optional[float] = None
  latitude: Optional[np.ndarray] = None
  longitude: Optional[np.ndarray] = None


@dataclasses.dataclass
class CombinedRegion:
  """regions.py:141-158."""
  regions: list = dataclasses.field(default_factory=list)


def _region_apply(region, x, w, lat, lon):
  """Region.apply on data `x` (..., lat, lon) with 2-D weights `w` (lat, lon).

  Returns (x, w, lat, lon) after the region (regions.py:40-158).  Weights are
  carried as a dense (lat, lon) array, which is what xarray broadcasting
  produces inside `weighted().mean` anyway.
  """
  if isinstance(region, SliceRegion):
    lats = region.lat_slice if isinstance(region.lat_slice, list) else [
        region.lat_slice]
    lons = region.lon_slice if isinstance(region.lon_slice, list) else [
        region.lon_slice]
    # regions.py:79-84: concat of label slices (no dedup)
    ilat = np.concatenate([_label_slice_indices(lat, s) for s in lats])
    ilon = np.concatenate([_label_slice_indices(lon, s) for s in lons])
    x = x[..., ilat, :][..., :, ilon]
    w = w[ilat, :][:, ilon]
    return x, w, lat[ilat], lon[ilon]
  if isinstance(region, ExtraTropicalRegion):
    region_weights = (np.abs(lat) >= 20).astype(float)  # regions.py:108
    return x, w * region_weights[:, None], lat, lon
  if isinstance(region, LandRegion):
    land = np.asarray(region.land_sea_mask)
    if region.latitude is not None:
      # xarray aligns `weights * land_weights` by coordinate label
      # (regions.py:138); after a SliceRegion the data grid is a subset
      ilat = np.array([int(np.nonzero(region.latitude == v)[0][0])
                       for v in lat])
      ilon = np.array([int(np.nonzero(region.longitude == v)[0][0])
                       for v in lon])
      land = land[ilat][:, ilon]
    if land.shape != (lat.size, lon.size):
      raise ValueError("oracle LandRegion needs a full (lat, lon) mask")
    if region.threshold is not None:
      land = (land > region.threshold).astype(float)  # regions.py:136-137
    return x, w * land, lat, lon
  if isinstance(region, CombinedRegion):
    for r in region.regions:  # regions.py:155-157
      x, w, lat, lon = _region_apply(r, x, w, lat, lon)
    return x, w, lat, lon
  raise TypeError(f"unknown region {region!r}")


# ----------------------------------------------------------------------------
# Weighted spatial mean -- metrics.py:141-172 + xarray Weighted._weighted_mean
# ----------------------------------------------------------------------------
def _to_lat_lon_last(x: np.ndarray, dims: Sequence[str]):
  dims = tuple(dims)
  ilat, ilon = dims.index(LAT), dims.index(LON)
  rest = [i for i in range(len(dims)) if i not in (ilat, ilon)]
  xt = np.transpose(x, rest + [ilat, ilon])
  return xt, tuple(dims[i] for i in rest)


def spatial_average(x, dims, lat, lon, region=None, skipna=False):
  """metrics.py:141-163.  Returns (result, out_dims); result is float64.

  xarray semantics restated (xarray/core/weighted.py `_weighted_mean`,
  `_sum_of_weights`, `_reduce`):
    sum  = dot(x.fillna(0) if skipna else x, w)
    sow  = dot(notnull(x), w)          # ALWAYS masked; sow == 0 -> NaN
    mean = sum / sow
  """
  lat = np.asarray(lat)
  lon = np.asarray(lon)
  xt, out_dims = _to_lat_lon_last(np.asarray(x), dims)
  w = np.broadcast_to(get_lat_weights(lat)[:, None], (lat.size, lon.size))
  if region is not None:
    xt, w, lat, lon = _region_apply(region, xt, w, lat, lon)
    xt = np.where(w > 0, xt, 0)  # metrics.py:160
  mask = ~np.isnan(xt)
  xs = np.where(mask, xt, 0) if skipna else xt
  with np.errstate(invalid="ignore", over="ignore"):
    num = np.einsum("...ij,ij->...", xs.astype(np.float64), w)
    den = np.einsum("...ij,ij->...", mask.astype(np.float64), w)
  den = np.where(den != 0.0, den, np.nan)
  with np.errstate(invalid="ignore", divide="ignore"):
    return num / den, out_dims


def spatial_average_l2_norm(x, dims, lat, lon, region=None, skipna=False):
  # metrics.py:166-172
  r, d = spatial_average(np.asarray(x) ** 2, dims, lat, lon, region, skipna)
  with np.errstate(invalid="ignore"):
    return np.sqrt(r), d


# ----------------------------------------------------------------------------
# Named-dim broadcasting (what xarray arithmetic does between two operands)
# ----------------------------------------------------------------------------
def align(a, adims, b, bdims):
  """Broadcast two named arrays against each other (xarray rule: result dims =
  dims of `a` in order, then dims only in `b`)."""
  adims, bdims = tuple(adims), tuple(bdims)
  out = list(adims) + [d for d in bdims if d not in adims]

  def expand(x, xd):
    x = np.asarray(x)
    perm = [xd.index(d) for d in out if d in xd]
    x = np.transpose(x, perm)
    shape = [slice(None) if d in xd else None for d in out]
    return x[tuple(shape)]

  return expand(a, adims), expand(b, bdims), tuple(out)


def time_mean(x, dims, skipna=False, avg_dim=None):
  """Metric.compute's `.mean(avg_dim, skipna=skipna)` -- metrics.py:117-138."""
  dims = tuple(dims)
  if avg_dim is None:
    avg_dim = "time" if "time" in dims else "init_time"
  ax = dims.index(avg_dim)
  with np.errstate(invalid="ignore"):
    import warnings
    with warnings.catch_warnings():
      warnings.simplefilter("ignore", RuntimeWarning)
      r = np.nanmean(x, axis=ax) if skipna else np.mean(x, axis=ax)
  return r, tuple(d for d in dims if d != avg_dim)


# ----------------------------------------------------------------------------
# Deterministic metrics -- metrics.py:175-414
# ----------------------------------------------------------------------------
def mse(f, fdims, t, tdims, lat, lon, region=None, skipna=False):
  # metrics.py:283-292
  fa, ta, d = align(f, fdims, t, tdims)
  return spatial_average((fa - ta) ** 2, d, lat, lon, region, skipna)


def rmse_sqrt_before_time_avg(f, fdims, t, tdims, lat, lon, region=None,
                              skipna=False):
  # metrics.py:251-260
  fa, ta, d = align(f, fdims, t, tdims)
  return spatial_average_l2_norm(fa - ta, d, lat, lon, region, skipna)


def mae(f, fdims, t, tdims, lat, lon, region=None, skipna=False):
  # metrics.py:323-330
  fa, ta, d = align(f, fdims, t, tdims)
  return spatial_average(np.abs(fa - ta), d, lat, lon, region, skipna)


def bias(f, fdims, t, tdims, lat, lon, region=None, skipna=False):
  # metrics.py:352-359
  fa, ta, d = align(f, fdims, t, tdims)
  return spatial_average(fa - ta, d, lat, lon, region, skipna)


def wind_vector_mse(fu, fv, fdims, tu, tv, tdims, lat, lon, region=None,
                    skipna=False):
  # metrics.py:189-202
  fua, tua, d = align(fu, fdims, tu, tdims)
  fva, tva, _ = align(fv, fdims, tv, tdims)
  du, dv = fua - tua, fva - tva
  return spatial_average(du ** 2 + dv ** 2, d, lat, lon, region, skipna)


def acc(f, fdims, t, tdims, c, cdims, lat, lon, region=None, skipna=False):
  """metrics.py:387-414.  `c` is the climatology ALREADY selected onto the
  forecast's (valid) times and levels (metrics.py:398-404 is label lookup)."""
  fa, ca, d1 = align(f, fdims, c, cdims)
  f_anom = fa - ca
  ta, ca2, d2 = align(t, tdims, c, cdims)
  t_anom = ta - ca2
  fa2, ta2, d = align(f_anom, d1, t_anom, d2)
  num, od = spatial_average(fa2 * ta2, d, lat, lon, region, skipna)
  ff, _ = spatial_average(f_anom ** 2, d1, lat, lon, region, skipna)
  tt, od2 = spatial_average(t_anom ** 2, d2, lat, lon, region, skipna)
  od1 = tuple(x for x in d1 if x not in (LAT, LON))
  ffa, tta, odp = align(ff, od1, tt, od2)
  numa, dena, odf = align(num, od, ffa * tta, odp)
  with np.errstate(invalid="ignore", divide="ignore"):
    return numa / np.sqrt(dena), odf


# ----------------------------------------------------------------------------
# Ensemble metrics -- metrics.py:532-846, 1161-1517
# ----------------------------------------------------------------------------
def _mean(x, axis, skipna):
  import warnings
  with warnings.catch_warnings():
    warnings.simplefilter("ignore", RuntimeWarning)
    with np.errstate(invalid="ignore"):
      return np.nanmean(x, axis=axis) if skipna else np.mean(x, axis=axis)


def _var(x, axis, skipna, ddof=1):
  import warnings
  with warnings.catch_warnings():
    warnings.simplefilter("ignore", RuntimeWarning)
    with np.errstate(invalid="ignore", divide="ignore"):
      if skipna:
        return np.nanvar(x, axis=axis, ddof=ddof)
      return np.var(x, axis=axis, ddof=ddof)


def rankdata(x: np.ndarray, axis: int) -> np.ndarray:
  """metrics.py:836-846 (ordinal ranks; NaN sorts last, np.argsort default)."""
  x = np.asarray(x)
  x = np.swapaxes(x, axis, -1)
  j = np.argsort(x, axis=-1)
  ordinal_ranks = np.broadcast_to(
      np.arange(1, x.shape[-1] + 1, dtype=int), x.shape)
  ordered_ranks = np.empty(j.shape, dtype=ordinal_ranks.dtype)
  np.put_along_axis(ordered_ranks, j, ordinal_ranks, axis=-1)
  return np.swapaxes(ordered_ranks, axis, -1)


def pointwise_crps_spread(f, fdims, ens_dim, skipna):
  # metrics.py:781-813
  fdims = tuple(fdims)
  ax = fdims.index(ens_dim)
  n = f.shape[ax]
  od = tuple(d for d in fdims if d != ens_dim)
  if n < 2:
    return np.zeros_like(np.take(f, 0, axis=ax)), od  # :788-789
  rank = rankdata(f, ax)
  return 2 * _mean((2 * rank - n - 1) * f, ax, skipna) / (n - 1), od


def pointwise_crps_skill(f, fdims, t, tdims, ens_dim, skipna):
  # metrics.py:816-824   abs(truth - forecast).mean(ensemble_dim)
  ta, fa, d = align(t, tdims, f, fdims)
  ax = d.index(ens_dim)
  return _mean(np.abs(ta - fa), ax, skipna), tuple(
      x for x in d if x != ens_dim)


def crps_spread(f, fdims, ens_dim, lat, lon, region=None, skipna=False):
  # metrics.py:682-694
  p, d = pointwise_crps_spread(f, fdims, ens_dim, skipna)
  return spatial_average(p, d, lat, lon, region, skipna)


def crps_skill(f, fdims, t, tdims, ens_dim, lat, lon, region=None,
               skipna=False):
  # metrics.py:701-715
  p, d = pointwise_crps_skill(f, fdims, t, tdims, ens_dim, skipna)
  return spatial_average(p, d, lat, lon, region, skipna)


def crps(f, fdims, t, tdims, ens_dim, lat, lon, region=None, skipna=False):
  # metrics.py:657-675
  sk, d1 = crps_skill(f, fdims, t, tdims, ens_dim, lat, lon, region, skipna)
  sp, d2 = crps_spread(f, fdims, ens_dim, lat, lon, region, skipna)
  a, b, d = align(sk, d1, sp, d2)
  return a - 0.5 * b, d


def ensemble_mean_mse(f, fdims, t, tdims, ens_dim, lat, lon, region=None,
                      skipna=False):
  # metrics.py:1319-1333
  fdims = tuple(fdims)
  m = _mean(f, fdims.index(ens_dim), skipna)
  md = tuple(x for x in fdims if x != ens_dim)
  ta, ma, d = align(t, tdims, m, md)
  return spatial_average((ta - ma) ** 2, d, lat, lon, region, skipna)


def ensemble_mean_rmse_sqrt_before_time_avg(f, fdims, t, tdims, ens_dim, lat,
                                            lon, region=None, skipna=False):
  # metrics.py:1293-1307
  fdims = tuple(fdims)
  m = _mean(f, fdims.index(ens_dim), skipna)
  md = tuple(x for x in fdims if x != ens_dim)
  ta, ma, d = align(t, tdims, m, md)
  return spatial_average_l2_norm(ta - ma, d, lat, lon, region, skipna)


def ensemble_variance(f, fdims, ens_dim, lat, lon, region=None, skipna=False):
  # metrics.py:1217-1241
  fdims = tuple(fdims)
  ax = fdims.index(ens_dim)
  od = tuple(x for x in fdims if x != ens_dim)
  if f.shape[ax] == 1:
    r, d = spatial_average(f, fdims, lat, lon, region, skipna)
    r = _mean(r, d.index(ens_dim), skipna)
    return np.zeros_like(r), tuple(x for x in d if x != ens_dim)
  return spatial_average(_var(f, ax, skipna), od, lat, lon, region, skipna)


def ensemble_stddev_sqrt_before_time_avg(f, fdims, ens_dim, lat, lon,
                                         region=None, skipna=False):
  # metrics.py:1185-1210
  fdims = tuple(fdims)
  ax = fdims.index(ens_dim)
  od = tuple(x for x in fdims if x != ens_dim)
  if f.shape[ax] == 1:
    r, d = spatial_average(f, fdims, lat, lon, region, skipna)
    r = _mean(r, d.index(ens_dim), skipna)
    return np.zeros_like(r), tuple(x for x in d if x != ens_dim)
  with np.errstate(invalid="ignore"):
    std = np.sqrt(_var(f, ax, skipna))
  return spatial_average_l2_norm(std, od, lat, lon, region, skipna)


def debiased_ensemble_mean_mse(f, fdims, t, tdims, ens_dim, lat, lon,
                               region=None, skipna=False):
  # metrics.py:532-565, 1347-1363
  fdims = tuple(fdims)
  ax = fdims.index(ens_dim)
  n = f.shape[ax]
  md = tuple(x for x in fdims if x != ens_dim)
  m = _mean(f, ax, skipna)
  v = _var(f, ax, skipna)
  ta, ma, d = align(t, tdims, m, md)
  biased = (ta - ma) ** 2
  ba, va, d2 = align(biased, d, v, md)
  return spatial_average(ba - va / n, d2, lat, lon, region, skipna)


def energy_score_skill(f, fdims, t, tdims, ens_dim, lat, lon, region=None,
                       skipna=False):
  # metrics.py:1503-1517
  fa, ta, d = align(f, fdims, t, tdims)
  r, od = spatial_average_l2_norm(fa - ta, d, lat, lon, region, skipna)
  return _mean(r, od.index(ens_dim), skipna), tuple(
      x for x in od if x != ens_dim)


def energy_score_spread(f, fdims, ens_dim, lat, lon, region=None,
                        skipna=False):
  # metrics.py:1471-1496
  fdims = tuple(fdims)
  ax = fdims.index(ens_dim)
  n = f.shape[ax]
  if n == 1:
    r, d = spatial_average(f, fdims, lat, lon, region, skipna)
    r = _mean(r, d.index(ens_dim), skipna)
    return np.zeros_like(r), tuple(x for x in d if x != ens_dim)
  a = np.take(f, np.arange(0, n - 1), axis=ax)
  b = np.take(f, np.arange(1, n), axis=ax)
  r, od = spatial_average_l2_norm(a - b, fdims, lat, lon, region, skipna)
  return _mean(r, od.index(ens_dim), skipna), tuple(
      x for x in od if x != ens_dim)


def energy_score(f, fdims, t, tdims, ens_dim, lat, lon, region=None,
                 skipna=False):
  # metrics.py:1446-1464
  sk, d1 = energy_score_skill(f, fdims, t, tdims, ens_dim, lat, lon, region,
                              skipna)
  sp, d2 = energy_score_spread(f, fdims, ens_dim, lat, lon, region, skipna)
  a, b, d = align(sk, d1, sp, d2)
  return a - 0.5 * b, d


def crps_brute_force(f, fdims, t, tdims, ens_dim, lat, lon, skipna):
  """The reference's own O(M^2) cross-check, metrics_test.py:896-920."""
  fdims = tuple(fdims)
  n = f.shape[fdims.index(ens_dim)]
  ta, fa, d = align(t, tdims, f, fdims)
  r, od = spatial_average(np.abs(ta - fa), d, lat, lon, None, skipna)
  skill = _mean(r, od.index(ens_dim), skipna)
  odr = tuple(x for x in od if x != ens_dim)
  if n == 1:
    spread = np.zeros_like(skill)
  else:
    gd = tuple("dummy" if x == ens_dim else x for x in fdims)
    a, b, d2 = align(f, fdims, f, gd)
    r2, od2 = spatial_average(np.abs(a - b), d2, lat, lon, None, skipna)
    r2 = _mean(r2, od2.index(ens_dim), skipna)
    od2 = tuple(x for x in od2 if x != ens_dim)
    r2 = _mean(r2, od2.index("dummy"), skipna)
    od2 = tuple(x for x in od2 if x != "dummy")
    a, b, odr = align(skill, odr, r2 * (n / (n - 1)), od2)
    skill, spread = a, b
  return {"score": skill - 0.5 * spread, "spread": spread, "skill": skill}, odr


# ----------------------------------------------------------------------------
# Conservative regridding -- weatherbench2/regridding.py:297-536
# The reference runs this in JAX with x64 disabled => float32 everywhere.
# `dtype` selects the arithmetic type (np.float32 = reference behaviour).
# ----------------------------------------------------------------------------
def _rg_latitude_cell_bounds(x, include_poles=True):
  # regridding.py:302-309
  if include_poles:
    initial = np.array([-90], dtype=x.dtype)
    final = np.array([90], dtype=x.dtype)
  else:
    initial = x[:1] - (x[1] - x[0]) / 2
    final = x[-1:] + (x[-1] - x[-2]) / 2
  return np.concatenate([initial, (x[:-1] + x[1:]) / 2, final])


def _rg_latitude_area_from_bounds(lower, upper):
  # regridding.py:312-314
  return np.sin(np.deg2rad(upper)) - np.sin(np.deg2rad(lower))


def _rg_latitude_area(points, include_poles):
  # regridding.py:317-320
  b = _rg_latitude_cell_bounds(points, include_poles)
  return _rg_latitude_area_from_bounds(b[:-1], b[1:])


def _rg_latitude_overlap(src, tgt, src_poles, tgt_poles):
  # regridding.py:323-338
  sb = _rg_latitude_cell_bounds(src, src_poles)
  tb = _rg_latitude_cell_bounds(tgt, tgt_poles)
  upper = np.minimum(tb[1:, None], sb[None, 1:])
  lower = np.maximum(tb[:-1, None], sb[None, :-1])
  return (upper > lower) * _rg_latitude_area_from_bounds(lower, upper)


def conservative_latitude_weights(src, tgt, src_poles, tgt_poles,
                                  dtype=np.float32):
  # regridding.py:341-373
  src = np.asarray(src, dtype=dtype)
  tgt = np.asarray(tgt, dtype=dtype)
  _assert_increasing(src)
  _assert_increasing(tgt)
  overlap = _rg_latitude_overlap(src, tgt, src_poles, tgt_poles)
  coverage = np.sum(overlap, axis=1, keepdims=True)
  with np.errstate(invalid="ignore", divide="ignore"):
    weights = overlap / coverage
  if not src_poles:
    target_areas = _rg_latitude_area(tgt, tgt_poles)[:, None]
    is_covered = np.isclose(coverage, target_areas, rtol=1e-3)
    weights = np.where(is_covered, weights, np.nan)
  return weights.astype(dtype)


def align_phase_with(x, target, period):
  # regridding.py:376-395
  if period is None:
    return x
  shift_down = x > target + period / 2
  shift_up = x < target - period / 2
  return x + period * shift_up - period * shift_down


def _periodic_upper_bounds(x, period):
  # regridding.py:398-405
  if period is None:
    x_plus = np.concatenate([x[1:], x[-1:] + (x[-1] - x[-2])])
  else:
    x_plus = align_phase_with(np.roll(x, -1), x, period)
  return (x + x_plus) / 2


def _periodic_lower_bounds(x, period):
  # regridding.py:408-415
  if period is None:
    x_minus = np.concatenate([x[:1] - (x[1] - x[0]), x[:-1]])
  else:
    x_minus = align_phase_with(np.roll(x, +1), x, period)
  return (x_minus + x) / 2


def _periodic_upper_lower_bounds(x, period):
  # regridding.py:418-423
  if period is not None:
    x = x % period
  return _periodic_upper_bounds(x, period), _periodic_lower_bounds(x, period)


def _longitude_length(points, periodic):
  # regridding.py:426-429
  upper, lower = _periodic_upper_lower_bounds(points, 360 if periodic else None)
  return upper - lower


def _periodic_overlap(x0, x1, y0, y1, period):
  # regridding.py:432-438
  y0 = align_phase_with(y0, x0, period)
  y1 = align_phase_with(y1, x0, period)
  upper = np.minimum(x1, y1)
  lower = np.maximum(x0, y0)
  return np.maximum(upper - lower, 0)


def _longitude_overlap(first, second, first_periodic, second_periodic):
  # regridding.py:441-459
  fu, fl = _periodic_upper_lower_bounds(first, 360 if first_periodic else None)
  su, sl = _periodic_upper_lower_bounds(
      second, 360 if second_periodic else None)
  return _periodic_overlap(fl[:, None], fu[:, None], sl[None, :], su[None, :],
                           360)


def conservative_longitude_weights(src, tgt, src_periodic, tgt_periodic,
                                   dtype=np.float32):
  # regridding.py:462-499
  src = np.asarray(src, dtype=dtype)
  tgt = np.asarray(tgt, dtype=dtype)
  if len(tgt) < 3 and tgt_periodic:
    raise ValueError(
        "Need 3 or more target points else overlap is not well defined. Found"
        f" {len(tgt)}")
  _assert_increasing(src)
  _assert_increasing(tgt)
  overlap = _longitude_overlap(tgt, src, tgt_periodic, src_periodic)
  coverage = np.sum(overlap, axis=1, keepdims=True)
  with np.errstate(invalid="ignore", divide="ignore"):
    weights = overlap / coverage
  if not src_periodic:
    target_lengths = _longitude_length(tgt, tgt_periodic)[:, None]
    is_covered = np.isclose(coverage, target_lengths, rtol=1e-3)
    weights = np.where(is_covered, weights, np.nan)
  return weights.astype(dtype)


@dataclasses.dataclass(frozen=True, eq=False)
class Grid:
  """regridding.py:117-179."""
  longitudes: np.ndarray
  latitudes: np.ndarray
  periodic: bool = True
  includes_poles: bool = True

  def __post_init__(self):
    _assert_increasing(np.asarray(self.latitudes))  # regridding.py:137-138

  @property
  def shape(self):
    return (len(self.longitudes), len(self.latitudes))


def conservative_regrid(field, source: Grid, target: Grid, dtype=np.float32):
  """ConservativeRegridder.regrid_array == _nanmean, regridding.py:502-536.
  `field` has dims (..., lon, lat); arithmetic in `dtype` (reference: f32)."""
  lon_w = conservative_longitude_weights(
      source.longitudes, target.longitudes, source.periodic, target.periodic,
      dtype)
  lat_w = conservative_latitude_weights(
      source.latitudes, target.latitudes, source.includes_poles,
      target.includes_poles, dtype)
  field = np.asarray(field).astype(dtype)
  nulls = np.isnan(field)

  def _mean(x):  # regridding.py:505-526
    with np.errstate(invalid="ignore", over="ignore"):
      return np.einsum("ab,cd,...bd->...ac", lon_w, lat_w, x.astype(dtype),
                       optimize=True).astype(dtype)

  total = _mean(np.where(nulls, 0, field))
  count = _mean(np.logical_not(nulls))
  with np.errstate(invalid="ignore", divide="ignore"):
    return (total / count).astype(dtype)  # NaN if count == 0 (:534)


# ----------------------------------------------------------------------------
# Zonal energy spectrum -- weatherbench2/derived_variables.py:531-626
# ----------------------------------------------------------------------------
def circumference(lat):
  # derived_variables.py:578-581
  return np.cos(np.asarray(lat) * np.pi / 180) * (2 * np.pi * EARTH_RADIUS_M)


def lon_spacing_m(lat, lon):
  # derived_variables.py:583-590
  diffs = np.diff(np.asarray(lon))
  if np.max(np.abs(diffs - diffs[0])) > 1e-3:
    raise ValueError(f"Expected uniform longitude spacing. {lon=}")
  return circumference(lat) * diffs[0] / 360


def zonal_energy_spectrum(x, dims, lat, lon):
  """derived_variables.py:592-626.  Returns (spectrum, dims, frequency,
  wavelength); `longitude` is replaced by `zonal_wavenumber` as the LAST dim
  (apply_ufunc moves the core dim to the end)."""
  dims = tuple(dims)
  x = np.asarray(x)
  spacing = lon_spacing_m(lat, lon)
  ax = dims.index(LON)
  xm = np.moveaxis(x, ax, -1)
  out_dims = tuple(d for d in dims if d != LON) + ("zonal_wavenumber",)
  f_k = np.fft.rfft(xm, axis=-1, norm="forward")  # :597
  one_and_many_twos = np.concatenate(([1], [2] * (f_k.shape[-1] - 1)))  # :600
  spectrum = np.real(f_k * np.conj(f_k)) * one_and_many_twos
  base_frequency = np.fft.rfftfreq(len(lon))  # :614
  with np.errstate(divide="ignore"):
    frequency = base_frequency[:, None] / spacing[None, :]  # (k, lat)  :618
    wavelength = 1 / frequency  # :621
  # multiply by circumference, broadcast along latitude  (:626)
  ilat = out_dims.index(LAT)
  shape = [1] * spectrum.ndim
  shape[ilat] = len(lat)
  spectrum = spectrum * circumference(lat).reshape(shape)
  return spectrum, out_dims, frequency, wavelength


def zonal_energy_spectrum_latitude_mean(x, dims, lat, lon, lat_slice=None):
  """The north star's "weighted meridional reduction" after the rFFT, defined on
  the reference's own pieces: the get_lat_weights-weighted (metrics.py:40-60)
  latitude mean of ZonalEnergySpectrum.compute (derived_variables.py:592-626),
  optionally over a label-inclusive latitude band.  Returns (result, dims)."""
  spec, sd, _, _ = zonal_energy_spectrum(x, dims, lat, lon)
  lat = np.asarray(lat)
  w = get_lat_weights(lat)
  if lat_slice is not None:
    lo = -np.inf if lat_slice.start is None else lat_slice.start
    hi = np.inf if lat_slice.stop is None else lat_slice.stop
    w = w * ((lat >= lo) & (lat <= hi))
  ax = sd.index(LAT)
  shape = [1] * spec.ndim
  shape[ax] = lat.size
  out = (spec * w.reshape(shape)).sum(axis=ax) / w.sum()
  return out, tuple(d for d in sd if d != LAT)


def interpolate_spectral_frequencies(spectrum, frequency, frequencies=None):
  """derived_variables.py:629-682 with its third-party call made directly:
  xarray's DataArray.interp(method='linear') is scipy.interpolate.interp1d(
  kind='linear', bounds_error=False, fill_value=nan) along the coordinate.
  spectrum: (..., latitude, wavenumber); frequency: (wavenumber, latitude).
  Returns (result (..., latitude, frequency), frequencies)."""
  from scipy import interpolate  # pylint: disable=import-outside-toplevel
  spectrum = np.asarray(spectrum)
  frequency = np.asarray(frequency, dtype=np.float64)
  nk, nlat = frequency.shape
  if frequencies is None:  # :658-664
    freq_min = frequency.max(axis=1).min()
    freq_max = frequency.min(axis=1).max()
    frequencies = np.linspace(freq_min, freq_max, num=nk)
  frequencies = np.asarray(frequencies, dtype=np.float64)
  out = np.empty(spectrum.shape[:-1] + (frequencies.size,), dtype=np.float64)
  for i in range(nlat):
    f = interpolate.interp1d(frequency[:, i], spectrum[..., i, :], axis=-1,
                             kind='linear', bounds_error=False,
                             fill_value=np.nan, assume_sorted=True)
    out[..., i, :] = f(frequencies)
  return out, frequencies


def ensemble_mean(x, axis, skipna=False):
  """scripts/compute_ensemble_mean.py:131 -- xbeam.Mean(realization, skipna):
  xarray / NumPy mean of float32 data (float32 result)."""
  x = np.asarray(x)
  with np.errstate(invalid='ignore'):
    import warnings  # pylint: disable=import-outside-toplevel
    with warnings.catch_warnings():
      warnings.simplefilter('ignore', RuntimeWarning)
      return np.nanmean(x, axis=axis) if skipna else np.mean(x, axis=axis)


# ---------------------------------------------------------------------------
# Map-output ("Spatial*") metrics: no spatial averaging (metrics.py:304-374,
# 718-772, 1244-1266, 1366-1399); Metric.compute then averages over time
# (metrics.py:117-138).
# ---------------------------------------------------------------------------
def spatial_det_map(stat, f, fdims, t, tdims):
  """stat in {'bias', 'mse', 'mae'}: forecast - truth, squared, absolute."""
  fa, ta, d = align(f, fdims, t, tdims)
  diff = fa - ta
  if stat == "bias":
    return diff, d  # metrics.py:374
  if stat == "mse":
    return diff ** 2, d  # metrics.py:316
  if stat == "mae":
    return np.abs(diff), d  # metrics.py:345
  raise ValueError(stat)


def spatial_ens_maps(f, fdims, t, tdims, ens_dim, skipna):
  """Point-wise ensemble statistics {name: (map, dims)}."""
  fdims = tuple(fdims)
  ax = fdims.index(ens_dim)
  n = f.shape[ax]
  od = tuple(x for x in fdims if x != ens_dim)
  skill, sd = pointwise_crps_skill(f, fdims, t, tdims, ens_dim, skipna)
  spread, pd_ = pointwise_crps_spread(f, fdims, ens_dim, skipna)
  m = _mean(f, ax, skipna)
  ta, ma, d = align(t, tdims, m, od)
  mse = (ta - ma) ** 2  # metrics.py:1381
  if n == 1:
    var = np.zeros_like(m)  # metrics.py:1257-1264
    var_for_debias = _var(f, ax, skipna)
  else:
    var = _var(f, ax, skipna)  # metrics.py:1266
    var_for_debias = var
  ba, va, d2 = align(mse, d, var_for_debias, od)
  sa, pa, d3 = align(skill, sd, spread, pd_)
  return {
      "skill": (skill, sd), "spread": (spread, pd_), "mse": (mse, d),
      "variance": (var, od), "debiased": (ba - va / n, d2),
      "crps": (sa - 0.5 * pa, d3),  # metrics.py:729-739
  }


# ---------------------------------------------------------------------------
# Gaussian-forecast and threshold metrics -- metrics.py:849-1158, 1523-1891,
# thresholds.py:152-185.  Point-wise scores on arrays that already broadcast
# against each other; callers apply spatial_average / time_mean.
# ---------------------------------------------------------------------------
def gaussian_quantile_threshold(clim_mean, clim_std, quantile):
  """thresholds.py:182-184 (np.float64 scalar * float32 array -> float64)."""
  from scipy import stats
  return clim_mean + np.float64(stats.norm.ppf(quantile)) * np.asarray(
      clim_std, dtype=np.float64)


def gaussian_crps_pointwise(f, s, t):
  """metrics.py:889-899."""
  from scipy import stats
  with np.errstate(invalid="ignore", divide="ignore"):
    norm_diff = (f - t) / s
    return s * (norm_diff * (2 * stats.norm.cdf(norm_diff) - 1)
                + 2 * stats.norm.pdf(norm_diff) - 1 / np.sqrt(np.pi))


def gaussian_brier_pointwise(f, s, t, thr):
  """metrics.py:963-980."""
  from scipy import stats
  with np.errstate(invalid="ignore", divide="ignore"):
    truth_probability = np.where(t > thr, 1.0, 0.0)
    exceedance = 1 - stats.norm.cdf((thr - f) / s)
    return (exceedance - truth_probability) ** 2


def gaussian_ignorance_pointwise(f, s, t, thr):
  """metrics.py:1029-1049."""
  from scipy import stats
  with np.errstate(invalid="ignore", divide="ignore"):
    truth_probability = np.where(t > thr, 1.0, 0.0)
    cdf = stats.norm.cdf((thr - f) / s)
    return -np.where(truth_probability.astype(bool), np.log(1 - cdf),
                     np.log(cdf))


def gaussian_rps_part_pointwise(f, s, t, thr):
  """metrics.py:1098-1118."""
  from scipy import stats
  with np.errstate(invalid="ignore", divide="ignore"):
    truth_ecdf = np.where(t < thr, 1.0, 0.0)
    cdf = stats.norm.cdf((thr - f) / s)
    return (cdf - truth_ecdf) ** 2


def ens_brier_pointwise(x, t, thr, ax, debias, skipna):
  """metrics.py:1523-1560; x has the member axis `ax`, t / thr do not."""
  te, the = np.expand_dims(t, ax), np.expand_dims(thr, ax)
  truth_probability = np.where(np.isnan(t), np.nan, np.where(t > thr, 1.0, 0.0))
  forecast_probability = np.where(np.isnan(x), np.nan,
                                  np.where(x > the, 1.0, 0.0))
  del te
  mean = _mean(forecast_probability, ax, skipna)
  biased = (mean - truth_probability) ** 2
  if not debias:
    return biased
  var = _var(forecast_probability, ax, skipna)
  # metrics.py:562-565 (note: truth - mean, squared: same value)
  return biased - var / x.shape[ax]


def ens_ignorance_pointwise(x, t, thr, ax, skipna):
  """metrics.py:1713-1729."""
  truth_probability = np.where(t > thr, 1.0, 0.0)
  forecast_probability = np.where(x > np.expand_dims(thr, ax), 1.0, 0.0)
  p = _mean(forecast_probability, ax, skipna)
  with np.errstate(divide="ignore"):
    return -np.where(truth_probability.astype(bool), np.log(p), np.log(1 - p))


def ens_rps_part_pointwise(x, t, thr, ax, skipna):
  """metrics.py:1793-1803."""
  truth_ecdf = np.where(t < thr, 1.0, 0.0)
  forecast_ecdf = np.where(x < np.expand_dims(thr, ax), 1.0, 0.0)
  return (_mean(forecast_ecdf, ax, skipna) - truth_ecdf) ** 2


# ---------------------------------------------------------------------------
# Nearest-neighbour and bilinear regridding -- regridding.py:212-294.
# ---------------------------------------------------------------------------
def nearest_neighbor_indices(source: Grid, target: Grid) -> np.ndarray:
  """regridding.py:212-228 (same BallTree / haversine query)."""
  from sklearn import neighbors
  source_mesh = np.meshgrid(np.deg2rad(source.latitudes),
                            np.deg2rad(source.longitudes))
  target_mesh = np.meshgrid(np.deg2rad(target.latitudes),
                            np.deg2rad(target.longitudes))
  index_coords = np.stack([x.ravel() for x in source_mesh], axis=-1)
  query_coords = np.stack([x.ravel() for x in target_mesh], axis=-1)
  tree = neighbors.BallTree(index_coords, metric="haversine")
  return tree.query(query_coords, return_distance=False).squeeze(axis=-1)


def nearest_regrid(field, source: Grid, target: Grid):
  """NearestRegridder.regrid_array, regridding.py:231-247; (..., lon, lat)."""
  field = np.asarray(field)
  if field.shape[-2:] != source.shape:
    raise ValueError(f"expected {field.shape=} to match {source.shape=}")
  idx = nearest_neighbor_indices(source, target)
  flat = field.reshape(field.shape[:-2] + (-1,))
  return np.take(flat, idx, axis=-1).reshape(field.shape[:-2] + target.shape)


def bilinear_regrid(field, source: Grid, target: Grid):
  """BilinearRegridder.regrid_array, regridding.py:256-294.  jnp.interp has
  np.interp's semantics (left / right / period); evaluated here in float64."""
  field = np.asarray(field, dtype=np.float64)
  lead = field.shape[:-2]
  x = field.reshape((-1,) + field.shape[-2:])
  # latitude (regridding.py:262-274): clamp at the ends iff the source has poles
  kw = {} if source.includes_poles else dict(left=np.nan, right=np.nan)
  lat_out = np.empty(x.shape[:2] + (len(target.latitudes),))
  for n in range(x.shape[0]):
    for b in range(x.shape[1]):
      lat_out[n, b] = np.interp(target.latitudes, source.latitudes, x[n, b],
                                **kw)
  # longitude (:276-292): periodic wrap-around or NaN outside
  kw = dict(period=360) if source.periodic else dict(left=np.nan, right=np.nan)
  out = np.empty((x.shape[0], len(target.longitudes), len(target.latitudes)))
  for n in range(x.shape[0]):
    for c in range(lat_out.shape[2]):
      out[n, :, c] = np.interp(target.longitudes, source.longitudes,
                               lat_out[n, :, c], **kw)
  return out.reshape(lead + out.shape[1:])


# ---------------------------------------------------------------------------
# SEEPS -- metrics.py:417-528.
# ---------------------------------------------------------------------------
def seeps_pointwise(f, t, wet_f, wet_t, p1, dry_threshold_mm=0.25, min_p1=0.1,
                    max_p1=0.85, dry_threshold=None):
  """SpatialSEEPS.compute_chunk on arrays that broadcast against each other:
  f / t precipitation, wet_f / wet_t the climatological wet threshold at their
  valid times, p1 the mean dry fraction.  Every operation runs in NumPy's
  promoted dtype, as in the reference: the Python-float thresholds are weak
  scalars, rounded to the dtype of the array they meet.  `dry_threshold` (in
  metres) replaces dry_threshold_mm / 1000 when given."""
  if dry_threshold is None:
    dry_threshold = dry_threshold_mm / 1000.0
  dry_threshold, min_p1, max_p1 = (float(dry_threshold), float(min_p1),
                                    float(max_p1))

  def cats(x, wet):  # metrics.py:446-460
    dry = x < dry_threshold
    light = np.logical_and(x > dry_threshold, x < wet)
    heavy = x >= wet
    c = np.stack([dry, light, heavy]).astype(int).astype(float)
    return np.where(np.isnan(x)[None], np.nan, c)

  fc, tc = cats(f, wet_f), cats(t, wet_t)
  out = fc[:, None] * tc[None, :]  # [forecast_cat, truth_cat, ...]
  z = np.zeros_like(p1, dtype=np.float64)
  with np.errstate(divide="ignore", invalid="ignore"):
    matrix = 0.5 * np.stack([  # metrics.py:482-494
        np.stack([z, 1 / (1 - p1), 4 / (1 - p1)]),
        np.stack([1 / p1, z, 3 / (1 - p1)]),
        np.stack([1 / p1 + 3 / (2 + p1), 3 / (2 + p1), z])])
  extra = out.ndim - 2 - np.ndim(p1)  # p1 has the trailing (spatial) dims
  matrix = matrix.reshape(matrix.shape[:2] + (1,) * extra + matrix.shape[2:])
  result = (out * matrix).sum(axis=(0, 1))  # xr.dot: NaN propagates
  result = np.where(p1 < max_p1, result, np.nan)  # :503-504
  return np.where(p1 > min_p1, result, np.nan)


# ---------------------------------------------------------------------------
# RankHistogram -- metrics.py:1894-2042 (without the random tie-breaking noise:
# truth is prepended to the members and a STABLE argsort keeps it first among
# equal values; NaN sorts last).
# ---------------------------------------------------------------------------
def rank_histogram_one_hot(f, fdims, t, tdims, ens_dim, num_bins=None):
  fdims = tuple(fdims)
  ax = fdims.index(ens_dim)
  m = f.shape[ax]
  od = tuple(d for d in fdims if d != ens_dim)
  ta, fa0, d = align(t, tdims, np.take(f, 0, axis=ax), od)
  ta = np.broadcast_to(np.transpose(ta, [d.index(x) for x in od]),
                       np.take(f, 0, axis=ax).shape)
  combined = np.concatenate([np.expand_dims(ta, ax), f], axis=ax)  # :2000-2009
  order = np.argsort(combined, axis=ax, kind="stable")
  ranks = np.argmin(order, axis=ax)  # position of element 0 (truth), :2027
  default_bins = m + 1
  nb = default_bins if num_bins is None else num_bins
  if default_bins % nb:
    raise ValueError(f"Cannot bin data with ensemble_size={m} into {nb} bins")
  ranks = ranks // (default_bins // nb)  # :1950-1958
  return np.eye(nb)[ranks], od + ("bins",)


# ----------------------------------------------------------------------------
# Baseline forecasts built from climatology / observations --
# weatherbench2/evaluation.py:165-193, 450-472, 607-656; utils.py:47-70.
# Plain loops over time stamps (Python datetimes via pandas), one slab at a
# time: what xarray's vectorised `.sel` materialises.
# ----------------------------------------------------------------------------
def _stamp_fields(times):
  import pandas as pd  # local: only these helpers need calendar arithmetic
  idx = pd.DatetimeIndex(np.asarray(times).ravel())
  return (np.asarray(idx.year), np.asarray(idx.dayofyear),
          np.asarray(idx.hour))


def climatology_like_forecast(clim, clim_dims, dayofyear, hour, valid_times):
  """`climatology.sel(dayofyear=vt.dt.dayofyear, hour=vt.dt.hour)`
  (evaluation.py:452-457).  `clim_dims` must contain 'dayofyear' and may
  contain 'hour'; returns (array, dims) with valid_times' axes first (named
  'vt0', 'vt1', ...) followed by the remaining climatology dims."""
  vt = np.asarray(valid_times)
  _, doy, hr = _stamp_fields(vt)
  has_hour = "hour" in clim_dims
  rest = [d for d in clim_dims if d not in ("dayofyear", "hour")]
  lead = ["dayofyear"] + (["hour"] if has_hour else [])
  c = np.transpose(clim, [clim_dims.index(d) for d in lead + rest])
  doy_pos = {int(d): i for i, d in enumerate(np.asarray(dayofyear))}
  hour_pos = ({int(h): i for i, h in enumerate(np.asarray(hour))}
              if has_hour else None)
  out = np.empty((vt.size,) + c.shape[len(lead):], dtype=clim.dtype)
  for n in range(vt.size):
    slab = c[doy_pos[int(doy[n])]]
    if has_hour:
      slab = slab[hour_pos[int(hr[n])]]
    out[n] = slab
  out = out.reshape(vt.shape + out.shape[1:])
  return out, tuple(f"vt{i}" for i in range(vt.ndim)) + tuple(rest)


def persistence_like_forecast_by_init(obs, obs_times, init_times, n_lead):
  """`truth.sel(time=init_time).expand_dims(lead_time=...)`
  (evaluation.py:644-651): array (init_time, lead_time, ...)."""
  pos = {np.datetime64(t, "ns"): i for i, t in enumerate(np.asarray(obs_times))}
  rows = [obs[pos[np.datetime64(t, "ns")]] for t in np.asarray(init_times)]
  at_init = np.stack(rows)
  return np.repeat(at_init[:, None], n_lead, axis=1)


def persistence_like_forecast_by_valid(obs, obs_times, times, leads):
  """evaluation.py:165-193: valid times from `times[0] + max(leads)` on; the
  observation at `valid time - lead` for every (time, lead).  Returns
  (kept_times, array (time, lead_time, ...))."""
  times = np.asarray(times)
  leads = np.asarray(leads)
  kept = times[times >= times[0] + leads.max()]
  pos = {np.datetime64(t, "ns"): i for i, t in enumerate(np.asarray(obs_times))}
  out = np.stack([np.stack([obs[pos[np.datetime64(t - l, "ns")]]
                            for l in leads]) for t in kept])
  return kept, out


def probabilistic_climatology(truth, times, start_year, end_year,
                              hour_interval):
  """utils.py:47-70: years stacked as members.  `truth` has time first.
  Returns (hours, dayofyear labels, array (hour, number, dayofyear, ...)) with
  NaN where a year has no value for that day (e.g. day 366)."""
  year, doy, hr = _stamp_fields(times)
  hours = list(range(0, 24, hour_interval))
  years = list(range(start_year, end_year + 1))
  wanted = [(y in years) and (h in hours) for y, h in zip(year, hr)]
  days = sorted({int(d) for d, w in zip(doy, wanted) if w})
  out = np.full((len(hours), len(years), len(days)) + truth.shape[1:], np.nan,
                dtype=truth.dtype)
  for n in range(len(year)):
    if wanted[n]:
      out[hours.index(int(hr[n])), years.index(int(year[n])),
          days.index(int(doy[n]))] = truth[n]
  return np.array(hours), np.array(days), out

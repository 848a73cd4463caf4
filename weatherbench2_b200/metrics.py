"""Evaluation metrics -- the operator classes of weatherbench2/metrics.py with
the arithmetic moved into hand-written sm_90a kernels (libwb2b200.so).

Same class names, constructor fields, `compute_chunk(forecast, truth, region,
skipna)` / `compute(...)` signatures, output structure and error behaviour as
the reference (weatherbench2/metrics.py:84-138).  Differences are internal:

  * the chunk is never copied or re-read per metric / region: one kernel pass
    yields every weighted sum (see csrc/det_metrics.cu, csrc/ens_metrics.cu);
  * inside `batch(...)` (used by evaluation._metric_and_region_loop) the first
    metric that touches a (forecast, truth) pair computes the sums for ALL
    regions and metric families of the eval config; later metric x region
    calls are served from that result.

Inputs are `xarray_lite.Dataset` objects (or real `xr.Dataset` when xarray is
installed); variable data may be NumPy arrays or CUDA torch tensors.
There is no CPU fallback: without the CUDA library the calls raise.
"""
from __future__ import annotations

import contextlib
import dataclasses
import threading
import typing as t

import numpy as np
import pandas as pd

from weatherbench2_b200 import _lib
from weatherbench2_b200 import _spatial as sp
from weatherbench2_b200 import xarray_lite as xl
from weatherbench2_b200.regions import Region

REALIZATION = 'realization'
LAT, LON = sp.LAT, sp.LON


@xl.boundary
def get_lat_weights(ds) -> xl.DataArray:
  """Latitude/area weights from the dataset's latitude coordinate
  (weatherbench2/metrics.py:55-60)."""
  lat = ds['latitude'].values if 'latitude' in ds else ds.latitude.values
  w = sp.lat_weights(lat)
  return xl.DataArray(w, ('latitude',), {'latitude': lat})


# ------------------------------------------------------------------------------
# Batched execution state
# ------------------------------------------------------------------------------
class _Batch(threading.local):
  def __init__(self):
    self.active = False
    self.regions: list = []
    self.climatology = None
    self.cache: dict = {}
    self.cell_cache: dict = {}


_batch = _Batch()
_global_cell_cache: dict = {}


@contextlib.contextmanager
def batch(regions: t.Optional[t.Sequence] = None, climatology=None):
  """Within this context the first spatial-sum request on a (forecast, truth)
  pair is evaluated for every region in `regions` (and with `climatology`, so
  that ACC shares the pass with MSE/MAE/Bias) and cached."""
  prev = (_batch.active, _batch.regions, _batch.climatology, _batch.cache)
  _batch.active = True
  _batch.regions = list(regions) if regions is not None else [None]
  _batch.climatology = climatology
  _batch.cache = {}
  try:
    yield
  finally:
    _batch.active, _batch.regions, _batch.climatology, _batch.cache = prev


def _region_index(region, regions) -> int:
  for i, r in enumerate(regions):
    if r is region:
      return i
  return -1


def _batch_index(region) -> int:
  """Index of `region` among the regions of the active `batch()`; -1 outside
  a batch or for another region."""
  return _region_index(region, _batch.regions) if _batch.active else -1


def _batch_cached(key, keep, compute):
  """`compute()`, evaluated once per `key` inside the active `batch()`.  The
  cache entry holds `keep` alive: the objects whose ids make up the key."""
  if key not in _batch.cache:
    _batch.cache[key] = (compute(), keep)
  return _batch.cache[key][0]


def _region_request(key, keep, compute, region):
  """(result, index of `region` in it): `compute(regions)` for all regions of
  the active `batch()`, cached under `key`, when `region` is one of them;
  else `compute([region])`."""
  ri = _batch_index(region)
  if ri < 0:
    return compute([region]), 0
  return _batch_cached(key, keep, lambda: compute(_batch.regions)), ri


def _context() -> _lib.Context:
  return _lib.default_context()


# ------------------------------------------------------------------------------
# Helpers shared by all metrics
# ------------------------------------------------------------------------------
def _common_vars(forecast: xl.Dataset, truth: xl.Dataset) -> list[str]:
  # Dataset arithmetic is an inner join on data variables (metrics.py:291)
  return [k for k in forecast.keys() if k in truth.keys()]


def _lat_lon(ds: xl.Dataset):
  lat = np.asarray(ds['latitude'].values)
  lon = np.asarray(ds['longitude'].values)
  sp.lat_weights(lat)  # same ValueError as metrics.py:35-37 via :48
  return lat, lon


def _paired_operands(forecast: xl.Dataset, truth: xl.Dataset,
                     dtype: t.Optional[np.dtype] = None):
  """Yields (name, f_da, t_da, f_op, t_op) for every variable of both datasets
  that has latitude and longitude dims: forecast and truth aligned by label
  (xarray arithmetic joins shared dimensions, inner join), the forecast
  operand in `dtype` (None: its own float type), the truth in the forecast
  operand's layout and dtype."""
  for name in _common_vars(forecast, truth):
    f_da, t_da = forecast[name], truth[name]
    if LAT not in f_da.dims or LON not in f_da.dims:
      continue
    f_da, t_da = xl.align_inner(f_da, t_da)
    f_op = sp.prepare_operand(f_da, None, dtype)
    t_op = sp.prepare_operand(t_da, f_op.layout, f_op.dtype)
    yield name, f_da, t_da, f_op, t_op


def _result_coords(out_dims, *sources: xl.DataArray) -> dict:
  coords = {}
  for s in sources:
    if s is None:
      continue
    for k, c in s.coords.items():
      if k in (LAT, LON):
        continue
      if all(d in out_dims for d in c.dims) and k not in coords:
        coords[k] = c
  return coords


def _ratio(num: np.ndarray, den: np.ndarray) -> np.ndarray:
  """xarray weighted mean: sum / sum_of_weights, NaN where the weights sum to
  zero (xarray/core/weighted.py; weatherbench2/metrics.py:161-163)."""
  with np.errstate(invalid='ignore', divide='ignore'):
    return np.where(den != 0.0, num / np.where(den != 0.0, den, 1.0), np.nan)


def _group_key(op: sp.Operand):
  return (op.on_device, op.dtype.str, op.layout, op.nrow, op.ncol,
          op.row_stride)


# ------------------------------------------------------------------------------
# Climatology lookup (metrics.py:63-81, 398-404) as an offset table
# ------------------------------------------------------------------------------
def _get_climatology_chunk(climatology: xl.Dataset, truth: xl.Dataset
                           ) -> xl.Dataset:
  """metrics.py:63-81."""
  try:
    return climatology[list(truth.keys())]
  except KeyError as e:
    not_found = set(truth.keys()).difference(climatology.keys())
    clim_var_dict = {str(key) + '_mean': key for key in truth.keys()}
    not_found_means = set(clim_var_dict).difference(climatology.keys())
    if not_found and not_found_means:
      raise KeyError(
          f'Did not find {not_found} keys in climatology. Appending '
          "'mean' did not help.") from e
    return climatology[list(clim_var_dict.keys())].rename(clim_var_dict)


def _clim_operand(clim_da: xl.DataArray, forecast: xl.Dataset,
                  f_da: xl.DataArray, want_layout, want_dtype) -> sp.Operand:
  """Operand addressing the climatology slab of every forecast field:
  level lookup (metrics.py:399-400) and dayofyear / hour lookup of the valid
  time (metrics.py:401-404), folded into the offset table."""
  op = sp.prepare_operand(clim_da, want_layout, want_dtype)
  time_dim = 'valid_time' if 'init_time' in forecast.dims else 'time'
  vt = forecast[time_dim]
  index_maps = {}
  stamps = pd.DatetimeIndex(vt.values.ravel())
  if 'dayofyear' in op.outer_dims:
    doy = np.asarray(stamps.dayofyear).reshape(vt.shape)
    pos = xl._lookup(clim_da.coords['dayofyear'].values, doy.ravel())  # pylint: disable=protected-access
    index_maps['dayofyear'] = (vt.dims, pos.reshape(vt.shape))
  if 'hour' in op.outer_dims:
    hour = np.asarray(stamps.hour).reshape(vt.shape)
    pos = xl._lookup(clim_da.coords['hour'].values, hour.ravel())  # pylint: disable=protected-access
    index_maps['hour'] = (vt.dims, pos.reshape(vt.shape))
  if 'level' in op.outer_dims and 'level' in f_da.dims:
    pos = xl._lookup(clim_da.coords['level'].values,  # pylint: disable=protected-access
                     f_da.coords['level'].values)
    index_maps['level'] = (('level',), pos)
  return sp.gather_operand(op, index_maps) if index_maps else op


# ------------------------------------------------------------------------------
# K1 front end
# ------------------------------------------------------------------------------
def _det_stats(forecast: xl.Dataset, truth: xl.Dataset, climatology,
               regions: t.Sequence, skipna: bool) -> dict:
  """{var: (stats[..., R, 10], out_dims, coords)} for all common variables."""
  ctx = _context()
  lat, lon = _lat_lon(forecast)
  clim_chunk = None
  if climatology is not None:
    clim_chunk = _get_climatology_chunk(xl.from_xarray(climatology), truth)
  prepared = {}
  for name, f_da, t_da, f_op, t_op in _paired_operands(forecast, truth):
    if t_op.row_stride != f_op.row_stride or t_op.on_device != f_op.on_device:
      raise ValueError(
          f'{name}: forecast and truth must share memory space and row stride')
    c_op = None
    if clim_chunk is not None and name in clim_chunk.keys():
      c_op = _clim_operand(clim_chunk[name], forecast, f_da, f_op.layout,
                           f_op.dtype)
    prepared[name] = (f_op, t_op, c_op, f_da, t_da)
  out = {}
  groups: dict = {}
  for name, (f_op, t_op, c_op, _, _) in prepared.items():
    groups.setdefault((_group_key(f_op), c_op is not None), []).append(name)
  for (_, has_clim), members in groups.items():
    f_ops = [prepared[n][0] for n in members]
    t_ops = [prepared[n][1] for n in members]
    c_ops = [prepared[n][2] for n in members] if has_clim else None
    stats, dims_list, _ = sp.run_det_metrics(
        ctx, f_ops, t_ops, c_ops, lat, lon, regions, skipna,
        _global_cell_cache)
    for n, st, dims in zip(members, stats, dims_list):
      coords = _result_coords(dims, prepared[n][3], prepared[n][4])
      out[n] = (st, dims, coords)
  return out


def _det_request(forecast, truth, region, skipna, climatology=None) -> dict:
  """Per-variable stats [..., 10] for one region (served from the batch cache
  when possible)."""
  if climatology is None and _batch_index(region) >= 0:
    climatology = _batch.climatology
  res, ri = _region_request(
      ('det', id(forecast), id(truth), id(climatology), bool(skipna)),
      (forecast, truth, climatology),
      lambda regions: _det_stats(forecast, truth, climatology, regions,
                                 skipna), region)
  return {k: (st[..., ri, :], dims, coords)
          for k, (st, dims, coords) in res.items()}


def _dataset_from(results: dict, fn) -> xl.Dataset:
  out = xl.Dataset()
  for name, (st, dims, coords) in results.items():
    out[name] = xl.DataArray(fn(st), dims, coords, name)
  return out


# ------------------------------------------------------------------------------
# Metric classes
# ------------------------------------------------------------------------------
@dataclasses.dataclass
class Metric(xl.Boundary):
  """Base class for metrics (weatherbench2/metrics.py:84-138)."""

  _boundary_methods = ('compute', 'compute_chunk')

  def compute_chunk(self, forecast, truth, region: t.Optional[Region] = None,
                    skipna: bool = False):
    """Evaluate this metric on a temporal chunk of data (metrics.py:88-115)."""
    raise NotImplementedError

  def compute(self, forecast, truth, region: t.Optional[Region] = None,
              skipna: bool = False):
    """Evaluate on datasets with full temporal coverage (metrics.py:117-138)."""
    if 'time' in forecast.dims:
      avg_dim = 'time'
    elif 'init_time' in forecast.dims:
      avg_dim = 'init_time'
    else:
      raise ValueError(
          f'Forecast has neither valid_time or init_time dimension {forecast}')
    return self.compute_chunk(
        forecast, truth, region=region, skipna=skipna).mean(
            avg_dim, skipna=skipna)


def _zero_truth(ds: xl.Dataset) -> xl.Dataset:
  """A (lat, lon)-only dataset of zeros: `ds - 0` turns the Bias / MSE
  statistics of K1 into plain weighted means of `ds` / `ds**2`."""
  zeros = xl.Dataset(coords={k: c for k, c in ds.coords.items()
                             if k in (LAT, LON)})
  for k in ds.keys():
    v = ds[k]
    sp_dims = tuple(d for d in v.dims if d in (LAT, LON))
    shape = tuple(v.sizes[d] for d in sp_dims)
    if xl._is_torch(v.data):  # pylint: disable=protected-access
      z = v.data.new_zeros(shape)
    else:
      z = np.zeros(shape, dtype=v.dtype if v.dtype.kind == 'f' else np.float64)
    zeros[k] = xl.DataArray(z, sp_dims)
  return zeros


@xl.boundary
def _spatial_average(dataset, region: t.Optional[Region], skipna: bool):
  """Weighted spatial mean of an arbitrary (lat, lon) dataset
  (weatherbench2/metrics.py:141-163), evaluated on the GPU as the Bias
  statistic of (dataset - 0)."""
  res = _det_stats(dataset, _zero_truth(dataset), None, [region], skipna)
  return _dataset_from(res, lambda st: _ratio(st[..., 0, 2], st[..., 0, 6]))


@xl.boundary
def _spatial_average_l2_norm(dataset, region, skipna):
  """sqrt(spatial_average(ds**2)) (metrics.py:166-172)."""
  res = _det_stats(dataset, _zero_truth(dataset), None, [region], skipna)
  with np.errstate(invalid='ignore'):
    return _dataset_from(
        res, lambda st: np.sqrt(_ratio(st[..., 0, 0], st[..., 0, 6])))


def _wind_vector_stat(forecast, truth, u_name, v_name, region, skipna):
  """sum W (du^2 + dv^2) / sum W  -- WindVectorMSE (metrics.py:189-202)."""
  ctx = _context()
  lat, lon = _lat_lon(forecast)
  das = [forecast[u_name], forecast[v_name], truth[u_name], truth[v_name]]
  with sp.Staging(ctx) as stage:
    fu = sp.prepare_operand(das[0])
    ops = [fu] + [sp.prepare_operand(d, fu.layout, fu.dtype) for d in das[1:]]
    if not fu.on_device:
      # the vector kernel has no streaming host entry: stage contiguous copies
      ops = []
      for d in das:
        arr = np.ascontiguousarray(d.values)
        op = sp.prepare_operand(xl.DataArray(arr, d.dims),
                                ops[0].layout if ops else None,
                                ops[0].dtype if ops else None)
        dptr = stage.array(np.ascontiguousarray(op.data))
        ops.append(dataclasses.replace(op, addr=dptr, on_device=True))
      fu = ops[0]
    for op in ops[1:]:
      if _group_key(op) != _group_key(fu):
        raise ValueError('wind components must share dtype, layout and device')
    fu_op, fv_op, tu_op, tv_op = ops
    dims, shape = sp.broadcast_dims(fu_op, tu_op, fv_op, tv_op)
    base, tabs = sp.addressing(ops, dims, shape)
    dtype_code = _lib.F32 if fu.dtype == np.float32 else _lib.F64
    groups = sp.build_weights(ctx, lat, lon, [region], fu.layout,
                              fu.row_stride, _global_cell_cache)
    st = sp.run_region_groups(
        ctx, groups, (tabs[0].size, 1, _lib.DET_NSTAT), 1,
        lambda w, out: ctx.det_metrics_vector(base, base, base, base,
                                              dtype_code, *tabs, w, skipna,
                                              out))
  st = st.reshape(shape + (_lib.DET_NSTAT,))
  coords = _result_coords(dims, das[0], das[2])
  return xl.DataArray(_ratio(st[..., 0], st[..., 6]), dims, coords)


@dataclasses.dataclass
class WindVectorMSE(Metric):
  """Wind vector mean square error (metrics.py:175-202)."""

  u_name: str
  v_name: str
  vector_name: str

  def compute_chunk(self, forecast, truth, region=None, skipna=False):
    return _wind_vector_stat(forecast, truth, self.u_name, self.v_name, region,
                             skipna)


@dataclasses.dataclass
class WindVectorRMSESqrtBeforeTimeAvg(Metric):
  """Wind vector RMSE, sqrt before time averaging (metrics.py:205-233)."""

  u_name: str
  v_name: str
  vector_name: str

  def compute_chunk(self, forecast, truth, region=None, skipna=False):
    mse = WindVectorMSE(
        u_name=self.u_name, v_name=self.v_name, vector_name=self.vector_name
    ).compute_chunk(forecast, truth, region=region, skipna=skipna)
    return np.sqrt(mse)


@dataclasses.dataclass
class RMSESqrtBeforeTimeAvg(Metric):
  """Root mean squared error, sqrt before time averaging (metrics.py:236-269).
  """

  wind_vector_rmse: t.Optional[list] = None

  def compute_chunk(self, forecast, truth, region=None, skipna=False):
    res = _det_request(forecast, truth, region, skipna)
    with np.errstate(invalid='ignore'):
      results = _dataset_from(
          res, lambda st: np.sqrt(_ratio(st[..., 0], st[..., 6])))
    if self.wind_vector_rmse is not None:
      for wv in self.wind_vector_rmse:
        results[wv.vector_name] = wv.compute_chunk(
            forecast, truth, region=region, skipna=skipna)
    return results


@dataclasses.dataclass
class MSE(Metric):
  """Mean squared error (metrics.py:272-301)."""

  wind_vector_mse: t.Optional[list] = None

  def compute_chunk(self, forecast, truth, region=None, skipna=False):
    res = _det_request(forecast, truth, region, skipna)
    results = _dataset_from(res, lambda st: _ratio(st[..., 0], st[..., 6]))
    if self.wind_vector_mse is not None:
      for wv in self.wind_vector_mse:
        results[wv.vector_name] = wv.compute_chunk(
            forecast, truth, region=region, skipna=skipna)
    return results


@dataclasses.dataclass
class MAE(Metric):
  """Mean absolute error (metrics.py:319-330)."""

  def compute_chunk(self, forecast, truth, region=None, skipna=False):
    res = _det_request(forecast, truth, region, skipna)
    return _dataset_from(res, lambda st: _ratio(st[..., 1], st[..., 6]))


@dataclasses.dataclass
class Bias(Metric):
  """Bias (metrics.py:348-359)."""

  def compute_chunk(self, forecast, truth, region=None, skipna=False):
    res = _det_request(forecast, truth, region, skipna)
    return _dataset_from(res, lambda st: _ratio(st[..., 2], st[..., 6]))


def _map_coords(out_dims, *sources: xl.DataArray) -> dict:
  """Coordinates (latitude / longitude included) that survive in a map."""
  coords = {}
  for s in sources:
    for k, c in s.coords.items():
      if all(d in out_dims for d in c.dims) and k not in coords:
        coords[k] = c
  return coords


def _avg_dim(forecast) -> str:
  if 'time' in forecast.dims:
    return 'time'
  if 'init_time' in forecast.dims:
    return 'init_time'
  raise ValueError(
      f'Forecast has neither valid_time or init_time dimension {forecast}')


@dataclasses.dataclass
class _SpatialDetMetric(Metric):
  """Map-output metrics: K6 (`wb2_det_maps`) computes stat(f, t) per grid cell
  and, in `compute`, the time mean in the same pass, so the per-time maps are
  never materialised.  `region` is ignored like in the reference."""

  def _maps(self, forecast, truth, reduce_dim, skipna):
    ctx = _context()
    out = xl.Dataset()
    for name, f_da, t_da, f_op, t_op in _paired_operands(forecast, truth):
      maps, dims = sp.run_det_maps(ctx, f_op, t_op, self._STAT, reduce_dim,
                                   skipna)
      out[name] = xl.DataArray(maps, dims, _map_coords(dims, f_da, t_da), name)
    return out

  def compute_chunk(self, forecast, truth, region=None, skipna=False):
    del region, skipna  # ignored (metrics.py:315, 344, 373)
    return self._maps(forecast, truth, None, False)

  def compute(self, forecast, truth, region=None, skipna=False):
    """metrics.py:117-138 with the time mean fused into the kernel."""
    del region
    return self._maps(forecast, truth, _avg_dim(forecast), skipna)


@dataclasses.dataclass
class SpatialMSE(_SpatialDetMetric):
  """MSE without spatial averaging (metrics.py:304-316)."""
  _STAT = _lib.MAP_MSE


@dataclasses.dataclass
class SpatialMAE(_SpatialDetMetric):
  """MAE without spatial averaging (metrics.py:333-345)."""
  _STAT = _lib.MAP_MAE


@dataclasses.dataclass
class SpatialBias(_SpatialDetMetric):
  """Bias without spatial averaging (metrics.py:362-374)."""
  _STAT = _lib.MAP_BIAS


@dataclasses.dataclass
class ACC(Metric):
  """Anomaly correlation coefficient (metrics.py:377-414)."""

  climatology: t.Any = None

  def __hash__(self):
    return id(self)

  def compute_chunk(self, forecast, truth, region=None, skipna=False):
    clim = xl.from_xarray(self.climatology)
    # fail like the reference when variables are missing (metrics.py:73-77)
    _get_climatology_chunk(clim, truth)
    res = _det_request(forecast, truth, region, skipna, climatology=clim)

    def acc(st):
      cov = _ratio(st[..., 3], st[..., 7])
      ff = _ratio(st[..., 4], st[..., 8])
      tt = _ratio(st[..., 5], st[..., 9])
      with np.errstate(invalid='ignore', divide='ignore'):
        return cov / np.sqrt(ff * tt)

    return _dataset_from(res, acc)


# Ensemble metrics live in _ensemble.py (they need the helpers above).
from weatherbench2_b200._ensemble import (  # noqa: E402  pylint: disable=wrong-import-position
    CRPS, CRPSSkill, CRPSSpread, DebiasedEnsembleMeanMSE, EnergyScore,
    EnergyScoreSkill, EnergyScoreSpread, EnsembleMeanMSE,
    EnsembleMeanRMSESqrtBeforeTimeAvg, EnsembleMetric,
    EnsembleStddevSqrtBeforeTimeAvg, EnsembleVariance, SpatialCRPS,
    SpatialCRPSSkill, SpatialCRPSSpread, SpatialEnsembleMeanMSE,
    SpatialEnsembleVariance, DebiasedSpatialEnsembleMeanMSE, _get_n_ensemble)
# SEEPS (precipitation categories) lives in _seeps.py.
from weatherbench2_b200._seeps import SEEPS, SpatialSEEPS  # noqa: E402  pylint: disable=wrong-import-position
from weatherbench2_b200._rank_hist import RankHistogram, central_reliability  # noqa: E402  pylint: disable=wrong-import-position
# Gaussian-forecast and threshold metrics live in _thresholded.py.
from weatherbench2_b200._thresholded import (  # noqa: E402  pylint: disable=wrong-import-position
    DebiasedEnsembleBrierScore, EnsembleBrierScore, EnsembleIgnoranceScore,
    EnsembleRPS, GaussianBrierScore, GaussianCRPS, GaussianIgnoranceScore,
    GaussianRPS, GaussianVariance, SpatialDebiasedEnsembleBrierScore,
    SpatialEnsembleBrierScore, SpatialEnsembleIgnoranceScore,
    SpatialEnsembleRPS, ThresholdMetric)

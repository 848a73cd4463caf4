"""Gaussian-forecast and threshold ("binary event") metric operators -- same
classes as weatherbench2/metrics.py:849-1158, 1523-1891 -- on top of K7
(csrc/threshold_metrics.cu).

Imported into `weatherbench2_b200.metrics`; use them from there.
"""
from __future__ import annotations

import dataclasses
import typing as t

import numpy as np

from weatherbench2_b200 import _ensemble as ens
from weatherbench2_b200 import _spatial as sp
from weatherbench2_b200 import metrics as m
from weatherbench2_b200 import thresholds as thr_lib
from weatherbench2_b200 import xarray_lite as xl

# slots of the K7 output (include/wb2b200.h)
_BRIER, _DEBIASED, _IGNORANCE, _RPS = 0, 1, 2, 3
_GCRPS, _GVAR = 0, 1


def _gaussian_vars(forecast: xl.Dataset) -> list[str]:
  """Variables that come with a `<var>_std` companion (metrics.py:891-894)."""
  return [k for k in forecast.keys() if f'{k}_std' in forecast.keys()]


def _threshold_spec(thresholds: t.Sequence, truth: xl.Dataset, name: str,
                    like: xl.DataArray, layout: str):
  """Kernel description of a list of thresholds for one variable."""
  if not thresholds:
    raise ValueError('at least one threshold is required')
  parts = [th.kernel_operands(truth, name, like, layout) for th in thresholds]
  kinds = {p[0] for p in parts}
  if len(kinds) != 1:
    raise ValueError('all thresholds of one metric must be of the same class')
  if parts[0][0] == 'field':
    return 'field', [p[1] for p in parts]
  clims = {id(th.climatology) for th in thresholds}
  if len(clims) != 1:
    raise ValueError('GaussianQuantileThresholds of one metric must share '
                     'their climatology')
  return 'gaussian', parts[0][1], parts[0][2], [p[3] for p in parts]


def _quantile_coords(thresholds):
  return xl.Coord(('quantile',), np.asarray([th.quantile for th in thresholds],
                                            dtype=np.float64))


def _stats_to_dataset(res: dict, slot: int, quantile_coord, sum_quantile: bool,
                      attrs: dict) -> xl.Dataset:
  """{var: (stats[..., nq, 8], dims, coords)} -> Dataset of sum / weight sum,
  `quantile` leading like the reference's expand_dims + concat
  (metrics.py:953-959)."""
  out = xl.Dataset(attrs=attrs)
  for name, (st, dims, coords) in res.items():
    val = m._ratio(st[..., slot], st[..., 4 + slot])  # pylint: disable=protected-access
    val = np.moveaxis(val, -1, 0)  # quantile first
    if sum_quantile:
      # xarray's `.sum("quantile")` (metrics.py:1158, 1866) skips NaN terms
      # (skipna defaults to True for float data)
      out[name] = xl.DataArray(np.nansum(val, axis=0), dims, coords, name)
    elif quantile_coord is None:
      out[name] = xl.DataArray(val[0], dims, coords, name)
    else:
      c = dict(coords)
      c['quantile'] = quantile_coord
      out[name] = xl.DataArray(val, ('quantile',) + tuple(dims), c, name)
  return out


# ------------------------------------------------------------------------------
# Gaussian forecasts
# ------------------------------------------------------------------------------
def _gaussian_stats(forecast: xl.Dataset, truth: xl.Dataset, thresholds,
                    regions: t.Sequence, skipna: bool) -> dict:
  ctx = m._context()  # pylint: disable=protected-access
  lat, lon = m._lat_lon(forecast)  # pylint: disable=protected-access
  out = {}
  for name in _gaussian_vars(forecast):
    if name not in truth.keys():
      raise KeyError(name)
    f_da, s_da, t_da = forecast[name], forecast[f'{name}_std'], truth[name]
    f_da, t_da = xl.align_inner(f_da, t_da)
    s_da, _ = xl.align_inner(s_da, t_da)
    m_op = sp.prepare_operand(f_da, None, np.float32)
    s_op = sp.prepare_operand(s_da, m_op.layout, np.float32)
    t_op = sp.prepare_operand(t_da, m_op.layout, np.float32)
    spec = None
    if thresholds is not None:
      spec = _threshold_spec(thresholds, truth, name, t_da, m_op.layout)
    st, dims = sp.run_gaussian_metrics(
        ctx, m_op, s_op, t_op, spec, lat, lon, regions, skipna,
        m._global_cell_cache)  # pylint: disable=protected-access
    coords = m._result_coords(dims, f_da, t_da)  # pylint: disable=protected-access
    out[name] = (st, dims, coords)
  return out


def _gaussian_request(forecast, truth, thresholds, region, skipna) -> dict:
  res, ri = m._region_request(  # pylint: disable=protected-access
      ('gauss', id(forecast), id(truth), bool(skipna),
       None if thresholds is None else tuple(id(th) for th in thresholds)),
      (forecast, truth, thresholds),
      lambda regions: _gaussian_stats(forecast, truth, thresholds, regions,
                                      skipna), region)
  return {k: (st[..., ri, :], dims, coords)
          for k, (st, dims, coords) in res.items()}


@dataclasses.dataclass
class GaussianCRPS(m.Metric):
  """The analytical CRPS of a Gaussian forecast (metrics.py:849-899)."""

  def compute_chunk(self, forecast, truth, region=None, skipna=False):
    res = _gaussian_request(forecast, truth, None, region, skipna)
    return _stats_to_dataset(res, _GCRPS, None, False, {})


@dataclasses.dataclass
class GaussianVariance(m.Metric):
  """The variance of a Gaussian forecast (metrics.py:902-928)."""

  def compute_chunk(self, forecast, truth, region=None, skipna=False):
    res = _gaussian_request(forecast, truth, None, region, skipna)
    return _stats_to_dataset(res, _GVAR, None, False, {})


@dataclasses.dataclass
class ThresholdMetric(m.Metric):
  """Base class for metrics based on thresholds (metrics.py:931-959)."""

  thresholds: t.Sequence[thr_lib.Threshold] = ()

  def __hash__(self):
    return id(self)

  def _attrs(self) -> dict:
    return {'threshold_method': type(self.thresholds[0]).__name__}


class _GaussianThresholdMetric(ThresholdMetric):
  _SLOT = _BRIER
  _SUM = False

  def compute_chunk(self, forecast, truth, region=None, skipna=False):
    res = _gaussian_request(forecast, truth, list(self.thresholds), region,
                            skipna)
    ds = _stats_to_dataset(res, self._SLOT, _quantile_coords(self.thresholds),
                           self._SUM, self._attrs())
    return ds


@dataclasses.dataclass
class GaussianBrierScore(_GaussianThresholdMetric):
  """Brier score of a Gaussian forecast (metrics.py:961-1026)."""
  _SLOT = _BRIER

  def __hash__(self):
    return id(self)


@dataclasses.dataclass
class GaussianIgnoranceScore(_GaussianThresholdMetric):
  """Ignorance score of a Gaussian forecast (metrics.py:1029-1095)."""
  _SLOT = _IGNORANCE

  def __hash__(self):
    return id(self)


@dataclasses.dataclass
class GaussianRPS(_GaussianThresholdMetric):
  """Ranked probability score of a Gaussian forecast, summed over the
  thresholds (metrics.py:1098-1158)."""
  _SLOT = _RPS
  _SUM = True

  def __hash__(self):
    return id(self)


# ------------------------------------------------------------------------------
# Ensemble forecasts
# ------------------------------------------------------------------------------
def _ens_threshold_stats(forecast: xl.Dataset, truth: xl.Dataset, ens_dim: str,
                         thresholds, regions: t.Sequence, skipna: bool) -> dict:
  ctx = m._context()  # pylint: disable=protected-access
  lat, lon = m._lat_lon(forecast)  # pylint: disable=protected-access
  out = {}
  for name, f_da, t_da, x_op, t_op in m._paired_operands(  # pylint: disable=protected-access
      forecast, truth, np.float32):
    spec = _threshold_spec(thresholds, truth, name, t_da, x_op.layout)
    st, dims, _ = sp.run_ens_threshold_metrics(
        ctx, x_op, t_op, ens_dim, spec, lat, lon, regions, skipna,
        m._global_cell_cache)  # pylint: disable=protected-access
    coords = m._result_coords(dims, f_da, t_da)  # pylint: disable=protected-access
    coords.pop(ens_dim, None)
    out[name] = (st, dims, coords)
  return out


def _ens_threshold_request(forecast, truth, ens_dim, thresholds, region,
                           skipna) -> dict:
  res, ri = m._region_request(  # pylint: disable=protected-access
      ('ensthr', id(forecast), id(truth), ens_dim, bool(skipna),
       tuple(id(th) for th in thresholds)),
      (forecast, truth, thresholds),
      lambda regions: _ens_threshold_stats(forecast, truth, ens_dim,
                                           thresholds, regions, skipna),
      region)
  return {k: (st[..., ri, :], dims, coords)
          for k, (st, dims, coords) in res.items()}


@dataclasses.dataclass
class _EnsembleThresholdMetric(ens.EnsembleMetric, ThresholdMetric):
  _SLOT = _BRIER
  _SUM = False

  def compute_chunk(self, forecast, truth, region=None, skipna=False):
    ens._get_n_ensemble(forecast, self.ensemble_dim)  # pylint: disable=protected-access
    res = _ens_threshold_request(forecast, truth, self.ensemble_dim,
                                 list(self.thresholds), region, skipna)
    ds = _stats_to_dataset(res, self._SLOT, _quantile_coords(self.thresholds),
                           self._SUM, self._attrs())
    return ds


@dataclasses.dataclass
class EnsembleBrierScore(_EnsembleThresholdMetric):
  """Brier score of an ensemble forecast for binary thresholds
  (metrics.py:1562-1612)."""
  _SLOT = _BRIER

  def __hash__(self):
    return id(self)


@dataclasses.dataclass
class DebiasedEnsembleBrierScore(_EnsembleThresholdMetric):
  """Brier score minus the sample variance / n of the member probabilities
  (metrics.py:1640-1698)."""
  _SLOT = _DEBIASED

  def __hash__(self):
    return id(self)


@dataclasses.dataclass
class EnsembleIgnoranceScore(_EnsembleThresholdMetric):
  """Ignorance (logarithmic) score of an ensemble forecast
  (metrics.py:1713-1765)."""
  _SLOT = _IGNORANCE

  def __hash__(self):
    return id(self)


@dataclasses.dataclass
class EnsembleRPS(_EnsembleThresholdMetric):
  """Ranked probability score, summed over the thresholds
  (metrics.py:1793-1865)."""
  _SLOT = _RPS
  _SUM = True

  def __hash__(self):
    return id(self)


@dataclasses.dataclass
class _SpatialEnsembleThresholdMetric(_EnsembleThresholdMetric):
  """Map-output threshold metrics: `wb2_ens_threshold_maps` gives the per-time
  score maps (`compute_chunk`) or, in `compute`, their time mean in the same
  pass.  `region` is ignored like in the reference (spatial_agg=False)."""

  def _maps(self, forecast, truth, reduce_dim, skipna):
    ens._get_n_ensemble(forecast, self.ensemble_dim)  # pylint: disable=protected-access
    ctx = m._context()  # pylint: disable=protected-access
    thresholds = list(self.thresholds)
    out = xl.Dataset(attrs=self._attrs())
    for name, f_da, t_da, x_op, t_op in m._paired_operands(  # pylint: disable=protected-access
        forecast, truth, np.float32):
      spec = _threshold_spec(thresholds, truth, name, t_da, x_op.layout)
      maps, dims, _ = sp.run_ens_threshold_maps(
          ctx, x_op, t_op, self.ensemble_dim, spec, self._SLOT, reduce_dim,
          skipna)
      coords = m._map_coords(dims, f_da, t_da)  # pylint: disable=protected-access
      coords.pop(self.ensemble_dim, None)
      if self._SUM:  # metrics.py:1891 `.sum("quantile")`
        if xl._is_torch(maps):  # pylint: disable=protected-access
          total = maps.nansum(0)
        else:
          total = np.nansum(maps, axis=0)
        out[name] = xl.DataArray(total, dims, coords, name)
      else:
        coords['quantile'] = _quantile_coords(thresholds)
        out[name] = xl.DataArray(maps, ('quantile',) + tuple(dims), coords,
                                 name)
    return out

  def compute_chunk(self, forecast, truth, region=None, skipna=False):
    del region
    return self._maps(forecast, truth, None, skipna)

  def compute(self, forecast, truth, region=None, skipna=False):
    del region
    result = self._maps(forecast, truth, m._avg_dim(forecast), skipna)  # pylint: disable=protected-access
    return result.assign_attrs(ensemble_size=forecast.sizes[self.ensemble_dim])


@dataclasses.dataclass
class SpatialEnsembleBrierScore(_SpatialEnsembleThresholdMetric):
  """Spatial map of the ensemble Brier score (metrics.py:1615-1637)."""
  _SLOT = _BRIER

  def __hash__(self):
    return id(self)


@dataclasses.dataclass
class SpatialDebiasedEnsembleBrierScore(_SpatialEnsembleThresholdMetric):
  """Spatial map of the debiased ensemble Brier score (metrics.py:1701-1710)."""
  _SLOT = _DEBIASED

  def __hash__(self):
    return id(self)


@dataclasses.dataclass
class SpatialEnsembleIgnoranceScore(_SpatialEnsembleThresholdMetric):
  """Spatial map of the ensemble ignorance score (metrics.py:1768-1790)."""
  _SLOT = _IGNORANCE

  def __hash__(self):
    return id(self)


@dataclasses.dataclass
class SpatialEnsembleRPS(_SpatialEnsembleThresholdMetric):
  """Spatial map of the ensemble RPS, summed over thresholds
  (metrics.py:1868-1891)."""
  _SLOT = _RPS
  _SUM = True

  def __hash__(self):
    return id(self)

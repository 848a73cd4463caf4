"""Ensemble (probabilistic) metric operators -- same classes as
weatherbench2/metrics.py:585-715, 1161-1517 -- on top of K2
(csrc/ens_metrics.cu) and, for the energy score, K1.

Imported into `weatherbench2_b200.metrics`; use them from there.
"""
from __future__ import annotations

import dataclasses
import typing as t

import numpy as np

from weatherbench2_b200 import _lib
from weatherbench2_b200 import _spatial as sp
from weatherbench2_b200 import metrics as m
from weatherbench2_b200 import xarray_lite as xl

REALIZATION = 'realization'

# indices into the K2 output (include/wb2b200.h, WB2_ENS_NSTAT)
_SKILL, _SPREAD, _MSE, _VAR, _DEBIASED = 0, 1, 2, 3, 4


def _get_n_ensemble(ds, ensemble_dim: str,
                    expect_n_ensemble_at_least: int = 1) -> int:
  """Size of `ensemble_dim` (weatherbench2/metrics.py:568-582)."""
  if ensemble_dim not in ds.dims:
    raise ValueError(f'{ensemble_dim=} not found in {ds.dims=}')
  n_ensemble = ds.sizes[ensemble_dim]
  if n_ensemble < expect_n_ensemble_at_least:
    raise ValueError(
        f'{n_ensemble=} is less than expected size of '
        f'{expect_n_ensemble_at_least}')
  return n_ensemble


def _ens_stats(forecast: xl.Dataset, truth: xl.Dataset, ens_dim: str,
               regions: t.Sequence, skipna: bool) -> dict:
  """{var: (stats[..., R, 10], dims, coords, M)} from ONE pass over the
  ensemble (skill, spread, ens-mean SE, variance, debiased SE)."""
  ctx = m._context()  # pylint: disable=protected-access
  lat, lon = m._lat_lon(forecast)  # pylint: disable=protected-access
  out = {}
  groups: dict = {}
  prepared = {}
  # K2 computes in float32 (float64 inputs are rounded to float32 first)
  for name, f_da, t_da, x_op, t_op in m._paired_operands(  # pylint: disable=protected-access
      forecast, truth, np.float32):
    prepared[name] = (x_op, t_op, f_da, t_da)
    groups.setdefault(m._group_key(x_op), []).append(name)  # pylint: disable=protected-access
  for _, members in groups.items():
    stats, dims_list, _, ms = sp.run_ens_metrics(
        ctx, [prepared[n][0] for n in members],
        [prepared[n][1] for n in members], ens_dim, lat, lon, regions, skipna,
        m._global_cell_cache)  # pylint: disable=protected-access
    for n, st, dims, mm in zip(members, stats, dims_list, ms):
      coords = m._result_coords(dims, prepared[n][2], prepared[n][3])  # pylint: disable=protected-access
      coords.pop(ens_dim, None)
      out[n] = (st, dims, coords, mm)
  return out


def _ens_request(forecast, truth, ens_dim, region, skipna) -> dict:
  res, ri = m._region_request(  # pylint: disable=protected-access
      ('ens', id(forecast), id(truth), ens_dim, bool(skipna)),
      (forecast, truth),
      lambda regions: _ens_stats(forecast, truth, ens_dim, regions, skipna),
      region)
  return {k: (st[..., ri, :], dims, coords, mm)
          for k, (st, dims, coords, mm) in res.items()}


def _ens_dataset(results: dict, fn) -> xl.Dataset:
  out = xl.Dataset()
  for name, (st, dims, coords, mm) in results.items():
    out[name] = xl.DataArray(fn(st, mm), dims, coords, name)
  return out


def _mean_stat(idx):
  return lambda st, mm: m._ratio(st[..., idx], st[..., 5 + idx])  # pylint: disable=protected-access


@dataclasses.dataclass
class EnsembleMetric(m.Metric):
  """Ensemble metric base class (metrics.py:585-607)."""

  ensemble_dim: str = REALIZATION

  def _ensemble_slice(self, ds, slice_obj: slice):
    """Slice `ds` and reset coords to 0..n-1 (metrics.py:591-596)."""
    ds = ds.isel({self.ensemble_dim: slice_obj})
    return ds.assign_coords(
        {self.ensemble_dim: np.arange(ds.sizes[self.ensemble_dim])})

  def compute(self, forecast, truth, region=None, skipna=False):
    """Adds the `ensemble_size` attribute (metrics.py:598-607)."""
    result = super().compute(forecast, truth, region=region, skipna=skipna)
    return result.assign_attrs(ensemble_size=forecast.sizes[self.ensemble_dim])


@dataclasses.dataclass
class CRPSSkill(EnsembleMetric):
  """E|X - Y| (metrics.py:697-715)."""

  def compute_chunk(self, forecast, truth, region=None, skipna=False):
    _get_n_ensemble(forecast, self.ensemble_dim)
    res = _ens_request(forecast, truth, self.ensemble_dim, region, skipna)
    return _ens_dataset(res, _mean_stat(_SKILL))


@dataclasses.dataclass
class CRPSSpread(EnsembleMetric):
  """E|X - X'| (metrics.py:678-694; M < 2 -> zeros, :788-789)."""

  def compute_chunk(self, forecast, truth, region=None, skipna=False):
    _get_n_ensemble(forecast, self.ensemble_dim)
    res = _ens_request(forecast, truth, self.ensemble_dim, region, skipna)
    return _ens_dataset(res, _mean_stat(_SPREAD))


@dataclasses.dataclass
class CRPS(EnsembleMetric):
  """CRPS = skill - spread / 2, each spatially averaged first
  (metrics.py:610-675)."""

  def compute_chunk(self, forecast, truth, region=None, skipna=False):
    _get_n_ensemble(forecast, self.ensemble_dim)
    res = _ens_request(forecast, truth, self.ensemble_dim, region, skipna)
    fn = lambda st, mm: (_mean_stat(_SKILL)(st, mm) -
                         0.5 * _mean_stat(_SPREAD)(st, mm))
    return _ens_dataset(res, fn)


@dataclasses.dataclass
class EnsembleMeanMSE(EnsembleMetric):
  """MSE of the ensemble mean (metrics.py:1310-1333)."""

  def compute_chunk(self, forecast, truth, region=None, skipna=False):
    _get_n_ensemble(forecast, self.ensemble_dim)
    res = _ens_request(forecast, truth, self.ensemble_dim, region, skipna)
    return _ens_dataset(res, _mean_stat(_MSE))


@dataclasses.dataclass
class EnsembleMeanRMSESqrtBeforeTimeAvg(EnsembleMetric):
  """RMSE of the ensemble mean, sqrt before time averaging
  (metrics.py:1269-1307)."""

  def compute_chunk(self, forecast, truth, region=None, skipna=False):
    _get_n_ensemble(forecast, self.ensemble_dim)
    res = _ens_request(forecast, truth, self.ensemble_dim, region, skipna)
    with np.errstate(invalid='ignore'):
      fn = lambda st, mm: np.sqrt(_mean_stat(_MSE)(st, mm))
      return _ens_dataset(res, fn)


def _zeros_for_single_member(st, idx):
  # metrics.py:1196-1204 / 1228-1235: zeros_like(spatial mean of the member);
  # NaN-ness does not survive zeros_like.
  return np.zeros(st.shape[:-1], dtype=np.float64)


@dataclasses.dataclass
class EnsembleVariance(EnsembleMetric):
  """Spatial mean of the ddof=1 ensemble variance (metrics.py:1213-1241)."""

  def compute_chunk(self, forecast, truth, region=None, skipna=False):
    n_ensemble = _get_n_ensemble(forecast, self.ensemble_dim)
    res = _ens_request(forecast, truth, self.ensemble_dim, region, skipna)
    if n_ensemble == 1:
      fn = lambda st, mm: _zeros_for_single_member(st, _VAR)
    else:
      fn = _mean_stat(_VAR)
    return _ens_dataset(res, fn)


@dataclasses.dataclass
class EnsembleStddevSqrtBeforeTimeAvg(EnsembleMetric):
  """sqrt(spatial mean of the ensemble variance): the reference takes `std`
  and then the L2 norm squares it again (metrics.py:1185-1210)."""

  def compute_chunk(self, forecast, truth, region=None, skipna=False):
    n_ensemble = _get_n_ensemble(forecast, self.ensemble_dim)
    res = _ens_request(forecast, truth, self.ensemble_dim, region, skipna)
    if n_ensemble == 1:
      fn = lambda st, mm: _zeros_for_single_member(st, _VAR)
    else:
      def fn(st, mm):
        with np.errstate(invalid='ignore'):
          return np.sqrt(_mean_stat(_VAR)(st, mm))
    return _ens_dataset(res, fn)


@dataclasses.dataclass
class DebiasedEnsembleMeanMSE(EnsembleMetric):
  """(t - xbar)^2 - var / M, spatially averaged (metrics.py:532-565,
  1336-1363).  NaN for a single member, like the reference."""

  def compute_chunk(self, forecast, truth, region=None, skipna=False):
    _get_n_ensemble(forecast, self.ensemble_dim)
    res = _ens_request(forecast, truth, self.ensemble_dim, region, skipna)
    return _ens_dataset(res, _mean_stat(_DEBIASED))


# ------------------------------------------------------------------------------
# Energy score.  skipna=False: K3 (csrc/ens_energy.cu) reads every member once.
# skipna=True: per-member weighted L2 norms via K1 on member views.
# ------------------------------------------------------------------------------
def _member_mean(ds: xl.Dataset, ens_dim: str, skipna: bool) -> xl.Dataset:
  return ds.mean(ens_dim, skipna=skipna)


def _energy_k3(forecast: xl.Dataset, truth: xl.Dataset, ens_dim: str, region):
  """(skill, spread) Datasets from ONE pass over the ensemble (K3)."""
  ctx = m._context()  # pylint: disable=protected-access
  lat, lon = m._lat_lon(forecast)  # pylint: disable=protected-access
  skill, spread = xl.Dataset(), xl.Dataset()
  for name, f_da, t_da, x_op, t_op in m._paired_operands(  # pylint: disable=protected-access
      forecast, truth, np.float32):
    (st,), (dims,), (mm,) = sp.run_energy_score(
        ctx, [x_op], [t_op], ens_dim, lat, lon, [region],
        m._global_cell_cache)  # pylint: disable=protected-access
    st = st[..., 0, :, :]  # single region
    coords = m._result_coords(dims, f_da, t_da)  # pylint: disable=protected-access
    coords.pop(ens_dim, None)
    with np.errstate(invalid='ignore', divide='ignore'):
      sk = np.sqrt(m._ratio(st[..., 0, :], st[..., 2, :])).mean(axis=-1)  # pylint: disable=protected-access
      if mm > 1:
        sd = np.sqrt(m._ratio(st[..., 1, :mm - 1],  # pylint: disable=protected-access
                              st[..., 3, :mm - 1])).mean(axis=-1)
      else:
        sd = np.zeros(st.shape[:-2], dtype=np.float64)  # metrics.py:1481-1489
    skill[name] = xl.DataArray(sk, dims, coords, name)
    spread[name] = xl.DataArray(sd, dims, coords, name)
  return skill, spread


def _use_k3(forecast, ens_dim, skipna) -> bool:
  return (not skipna) and forecast.sizes[ens_dim] <= 64


@dataclasses.dataclass
class EnergyScoreSkill(EnsembleMetric):
  """mean_m sqrt(SA((x_m - t)^2)) (metrics.py:1499-1517)."""

  def compute_chunk(self, forecast, truth, region=None, skipna=False):
    _get_n_ensemble(forecast, self.ensemble_dim)
    if _use_k3(forecast, self.ensemble_dim, skipna):
      return _energy_k3(forecast, truth, self.ensemble_dim, region)[0]
    res = m._det_request(forecast, truth, region, skipna)  # pylint: disable=protected-access
    with np.errstate(invalid='ignore'):
      l2 = m._dataset_from(  # pylint: disable=protected-access
          res, lambda st: np.sqrt(m._ratio(st[..., 0], st[..., 6])))  # pylint: disable=protected-access
    return _member_mean(l2, self.ensemble_dim, skipna)


@dataclasses.dataclass
class EnergyScoreSpread(EnsembleMetric):
  """mean over the M-1 adjacent member pairs of sqrt(SA((x_m - x_{m+1})^2))
  (metrics.py:1467-1496); zeros for a single member."""

  def compute_chunk(self, forecast, truth, region=None, skipna=False):
    n_ensemble = _get_n_ensemble(forecast, self.ensemble_dim)
    if _use_k3(forecast, self.ensemble_dim, skipna):
      return _energy_k3(forecast, truth, self.ensemble_dim, region)[1]
    if n_ensemble == 1:
      res = m._det_request(forecast, m._zero_truth(forecast), region, skipna)  # pylint: disable=protected-access
      zeros = m._dataset_from(  # pylint: disable=protected-access
          res, lambda st: np.zeros(st.shape[:-1], dtype=np.float64))
      return _member_mean(zeros, self.ensemble_dim, skipna)
    a = self._ensemble_slice(forecast, slice(None, -1))  # views, no copies
    b = self._ensemble_slice(forecast, slice(1, None))
    res = m._det_stats(a, b, None, [region], skipna)  # pylint: disable=protected-access
    res = {k: (st[..., 0, :], dims, coords)
           for k, (st, dims, coords) in res.items()}
    with np.errstate(invalid='ignore'):
      l2 = m._dataset_from(  # pylint: disable=protected-access
          res, lambda st: np.sqrt(m._ratio(st[..., 0], st[..., 6])))  # pylint: disable=protected-access
    return _member_mean(l2, self.ensemble_dim, skipna)


@dataclasses.dataclass
class EnergyScore(EnsembleMetric):
  """ES = skill - spread / 2 (metrics.py:1402-1464)."""

  def compute_chunk(self, forecast, truth, region=None, skipna=False):
    _get_n_ensemble(forecast, self.ensemble_dim)
    if _use_k3(forecast, self.ensemble_dim, skipna):
      skill, spread = _energy_k3(forecast, truth, self.ensemble_dim, region)
      return skill - 0.5 * spread
    return EnergyScoreSkill(self.ensemble_dim).compute_chunk(
        forecast, truth, region=region, skipna=skipna
    ) - 0.5 * EnergyScoreSpread(self.ensemble_dim).compute_chunk(
        forecast, truth, region=region, skipna=skipna)


# ------------------------------------------------------------------------------
# Map-output ("Spatial*") ensemble metrics: K6e (csrc/ens_maps.cu)
# ------------------------------------------------------------------------------
_MAP_BITS = (_lib.ENS_SKILL, _lib.ENS_SPREAD, _lib.ENS_MEAN_SE,
             _lib.ENS_VARIANCE, _lib.ENS_DEBIASED, _lib.ENS_CRPS)
_ALL_MAPS = sum(_MAP_BITS)


def _ens_maps(forecast: xl.Dataset, truth: xl.Dataset, ens_dim: str,
              stat_mask: int, reduce_dim: t.Optional[str], skipna: bool) -> dict:
  """{var: (maps[nsel, ...], dims, coords, M)} for the selected statistics."""
  ctx = m._context()  # pylint: disable=protected-access
  out = {}
  for name, f_da, t_da, x_op, t_op in m._paired_operands(  # pylint: disable=protected-access
      forecast, truth, np.float32):
    maps, dims, mm = sp.run_ens_maps(ctx, x_op, t_op, ens_dim, stat_mask,
                                     reduce_dim, skipna)
    coords = m._map_coords(dims, f_da, t_da)  # pylint: disable=protected-access
    coords.pop(ens_dim, None)
    out[name] = (maps, dims, coords, mm)
  return out


def _ens_map_request(forecast, truth, ens_dim, bit, reduce_dim, skipna):
  """One statistic's maps; inside `metrics.batch()` all six come from a single
  pass over the ensemble and are shared by the Spatial* metrics."""
  if m._batch.active:  # pylint: disable=protected-access
    res = m._batch_cached(  # pylint: disable=protected-access
        ('ensmap', id(forecast), id(truth), ens_dim, reduce_dim, bool(skipna)),
        (forecast, truth),
        lambda: _ens_maps(forecast, truth, ens_dim, _ALL_MAPS, reduce_dim,
                          skipna))
    sel = _MAP_BITS.index(bit)
  else:
    res, sel = _ens_maps(forecast, truth, ens_dim, bit, reduce_dim, skipna), 0
  out = xl.Dataset()
  for name, (maps, dims, coords, _) in res.items():
    out[name] = xl.DataArray(maps[sel], dims, coords, name)
  return out


@dataclasses.dataclass
class _SpatialEnsembleMetric(EnsembleMetric):
  """Base of the map-output ensemble metrics: `compute_chunk` gives the
  per-time maps, `compute` fuses the time mean into the kernel."""

  def _maps(self, forecast, truth, reduce_dim, skipna):
    n_ensemble = _get_n_ensemble(forecast, self.ensemble_dim)
    ds = _ens_map_request(forecast, truth, self.ensemble_dim, self._BIT,
                          reduce_dim, skipna)
    if n_ensemble == 1 and self._ZERO_FOR_SINGLE_MEMBER:
      # metrics.py:1257-1264: zeros_like(forecast).mean(ensemble_dim)
      for name in list(ds.keys()):
        da = ds[name]
        ds[name] = xl.DataArray(xl.zeros_like(da).data, da.dims, da.coords,
                                name)
    return ds

  def compute_chunk(self, forecast, truth, region=None, skipna=False):
    del region  # ignored, like the reference
    return self._maps(forecast, truth, None, skipna)

  def compute(self, forecast, truth, region=None, skipna=False):
    del region
    result = self._maps(forecast, truth, m._avg_dim(forecast), skipna)  # pylint: disable=protected-access
    return result.assign_attrs(ensemble_size=forecast.sizes[self.ensemble_dim])


@dataclasses.dataclass
class SpatialCRPS(_SpatialEnsembleMetric):
  """CRPS without spatial averaging (metrics.py:718-739)."""
  _BIT = _lib.ENS_CRPS
  _ZERO_FOR_SINGLE_MEMBER = False


@dataclasses.dataclass
class SpatialCRPSSpread(_SpatialEnsembleMetric):
  """CRPSSpread without spatial averaging (metrics.py:742-754)."""
  _BIT = _lib.ENS_SPREAD
  _ZERO_FOR_SINGLE_MEMBER = False


@dataclasses.dataclass
class SpatialCRPSSkill(_SpatialEnsembleMetric):
  """CRPSSkill without spatial averaging (metrics.py:757-772)."""
  _BIT = _lib.ENS_SKILL
  _ZERO_FOR_SINGLE_MEMBER = False


@dataclasses.dataclass
class SpatialEnsembleVariance(_SpatialEnsembleMetric):
  """Ensemble variance without spatial averaging (metrics.py:1244-1266)."""
  _BIT = _lib.ENS_VARIANCE
  _ZERO_FOR_SINGLE_MEMBER = True


@dataclasses.dataclass
class SpatialEnsembleMeanMSE(_SpatialEnsembleMetric):
  """Squared error of the ensemble mean per grid cell (metrics.py:1366-1381)."""
  _BIT = _lib.ENS_MEAN_SE
  _ZERO_FOR_SINGLE_MEMBER = False


@dataclasses.dataclass
class DebiasedSpatialEnsembleMeanMSE(_SpatialEnsembleMetric):
  """Debiased squared error of the ensemble mean per grid cell
  (metrics.py:1384-1399)."""
  _BIT = _lib.ENS_DEBIASED
  _ZERO_FOR_SINGLE_MEMBER = False

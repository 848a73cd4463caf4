"""Thresholding classes for discrete probabilistic metrics -- same classes as
weatherbench2/thresholds.py:92-197.

`Threshold.compute(truth)` materialises the threshold dataset exactly like the
reference (host NumPy; used by user code and tests).  The metric kernels do not
call it: `kernel_operands` describes the same selection as offset tables into
the climatology (day-of-year / hour / level / quantile lookups folded into the
table, like ACC's climatology), and for GaussianQuantileThreshold the
threshold `mean + ppf(q) * std` is evaluated inside the kernel in float64.
"""
from __future__ import annotations

import dataclasses
import typing as t

import numpy as np
import pandas as pd
from scipy import special

from weatherbench2_b200 import _spatial as sp
from weatherbench2_b200 import xarray_lite as xl


def _get_climatology_mean(climatology: xl.Dataset, variables: t.Sequence[str]
                          ) -> xl.Dataset:
  """thresholds.py:25-46."""
  try:
    return climatology[list(variables)]
  except KeyError as e:
    not_found = set(variables).difference(climatology.keys())
    clim_var_dict = {var + '_mean': var for var in variables}
    not_found_means = set(clim_var_dict).difference(climatology.keys())
    if not_found and not_found_means:
      raise KeyError(
          f'Did not find {not_found} keys in climatology. Appending '
          "'mean' did not help.") from e
    return climatology[list(clim_var_dict.keys())].rename(clim_var_dict)


def _get_climatology_std(climatology: xl.Dataset, variables: t.Sequence[str]
                         ) -> xl.Dataset:
  """thresholds.py:49-62."""
  clim_std_dict = {key + '_std': key for key in variables}
  try:
    return climatology[list(clim_std_dict.keys())].rename(clim_std_dict)
  except KeyError as e:
    not_found_stds = set(clim_std_dict).difference(climatology.keys())
    raise KeyError(
        f'Did not find {not_found_stds} keys in climatology.') from e


def _quantile_position(coord: np.ndarray, quantile: float, atol: float) -> int:
  """`.sel(quantile=q, method='nearest', tolerance=atol)` (thresholds.py:79-89)."""
  coord = np.asarray(coord, dtype=np.float64)
  pos = int(np.abs(coord - quantile).argmin())
  if not abs(coord[pos] - quantile) <= atol:
    raise KeyError(
        f'Did not find quantiles {quantile}+-{atol} in climatology.'
        ' Consider increasing the tolerance or recomputing the climatology.')
  return pos


def _get_climatology_quantile(climatology: xl.Dataset,
                              variables: t.Sequence[str]) -> xl.Dataset:
  """The `<var>_quantile` variables renamed to `<var>` (thresholds.py:65-78);
  the nearest-quantile selection happens in the callers."""
  clim_q_dict = {key + '_quantile': key for key in variables}
  try:
    return climatology[list(clim_q_dict.keys())].rename(clim_q_dict)
  except KeyError as e:
    not_found_qs = set(clim_q_dict).difference(climatology.keys())
    raise KeyError(f'Did not find {not_found_qs} keys in climatology.') from e


def _truth_time(truth: xl.Dataset):
  """(dims, timestamps) of the truth's valid time: the `time` coordinate the
  reference reads (thresholds.py:139, 173) -- 1-D, or 2-D (init_time,
  lead_time) after `truth.sel(time=forecast.valid_time)` where this package
  keeps it under `valid_time`."""
  for key in ('time', 'valid_time'):
    if key in truth.coords:
      c = truth.coords[key]
      return tuple(c.dims), np.asarray(c.values)
  raise KeyError('truth has neither a time nor a valid_time coordinate')


def _selection_maps(clim_da: xl.DataArray, truth: xl.Dataset,
                    like: xl.DataArray) -> dict:
  """index maps {clim_dim: (new_dims, positions)} of the day-of-year / hour /
  level lookups (thresholds.py:134-142, 168-176)."""
  del truth  # the variable's own (possibly label-aligned) time is what counts
  tdims, stamps = _truth_time(like)
  idx = pd.DatetimeIndex(stamps.ravel())
  maps = {}
  if 'level' in clim_da.dims and 'level' in like.dims:
    pos = xl._lookup(clim_da.coords['level'].values,  # pylint: disable=protected-access
                     like.coords['level'].values)
    maps['level'] = (('level',), pos)
  if 'dayofyear' in clim_da.dims:
    pos = xl._lookup(clim_da.coords['dayofyear'].values,  # pylint: disable=protected-access
                     np.asarray(idx.dayofyear))
    maps['dayofyear'] = (tdims, pos.reshape(stamps.shape))
  if 'hour' in clim_da.dims:
    pos = xl._lookup(clim_da.coords['hour'].values,  # pylint: disable=protected-access
                     np.asarray(idx.hour))
    maps['hour'] = (tdims, pos.reshape(stamps.shape))
  return maps


def _materialise(clim_da: xl.DataArray, maps: dict) -> xl.DataArray:
  """The selected climatology as an array (host gather)."""
  arr = np.asarray(clim_da.values)
  dims = list(clim_da.dims)
  # level first (keeps its dim), then the joint time lookup
  if 'level' in maps:
    ax = dims.index('level')
    arr = np.take(arr, maps['level'][1], axis=ax)
  time_keys = [k for k in ('dayofyear', 'hour') if k in maps]
  coords = {k: c for k, c in clim_da.coords.items()
            if k not in ('dayofyear', 'hour') and not (
                set(c.dims) & {'dayofyear', 'hour'})}
  if 'level' in maps and 'level' in coords:
    coords['level'] = xl.Coord(('level',), np.asarray(
        clim_da.coords['level'].values)[maps['level'][1]])
  if time_keys:
    tdims = maps[time_keys[0]][0]
    axes = [dims.index(k) for k in time_keys]
    arr = np.moveaxis(arr, axes, range(len(axes)))
    arr = arr[tuple(maps[k][1] for k in time_keys)]
    dims = list(tdims) + [d for d in dims if d not in time_keys]
  return xl.DataArray(arr, tuple(dims), coords, clim_da.name)


@dataclasses.dataclass
class Threshold(xl.Boundary):
  """Threshold for discrete probabilistic metric evaluation
  (thresholds.py:92-115)."""

  _boundary_methods = ('compute',)

  climatology: t.Any
  quantile: float

  def __hash__(self):
    return id(self)

  def compute(self, truth) -> xl.Dataset:
    raise NotImplementedError

  def kernel_operands(self, truth: xl.Dataset, name: str, like: xl.DataArray,
                      layout: str):
    """Describes this threshold for variable `name` to the kernels:
    ('field', operand) or ('gaussian', mean_operand, std_operand, z)."""
    raise NotImplementedError


@dataclasses.dataclass
class QuantileThreshold(Threshold):
  """Climatological quantile threshold (thresholds.py:118-149)."""

  def __hash__(self):
    return id(self)

  def compute(self, truth) -> xl.Dataset:
    clim = xl.from_xarray(self.climatology)
    variables = [str(k) for k in truth.keys()]
    clim_q = _get_climatology_quantile(clim, variables)
    out = xl.Dataset()
    for name in variables:
      da = clim_q[name]
      sel = _materialise(da, _selection_maps(da, truth, truth[name]))
      if 'quantile' in sel.dims:
        pos = _quantile_position(sel.coords['quantile'].values, self.quantile,
                                 0.01)
        sel = sel.isel(quantile=pos)
      out[name] = sel
    return out

  def kernel_operands(self, truth, name, like, layout):
    clim = xl.from_xarray(self.climatology)
    da = _get_climatology_quantile(clim, [name])[name]
    op = sp.prepare_operand(da, layout, np.float32)
    maps = _selection_maps(da, truth, like)
    if 'quantile' in da.dims:
      pos = _quantile_position(da.coords['quantile'].values, self.quantile,
                               0.01)
      maps['quantile'] = ((), np.asarray(pos, dtype=np.int64))
    return 'field', sp.gather_operand(op, maps)


@dataclasses.dataclass
class GaussianQuantileThreshold(Threshold):
  """Quantile of a Gaussian fitted to the climatology: mean + ppf(q) * std
  (thresholds.py:152-185)."""

  def __hash__(self):
    return id(self)

  def z(self) -> float:
    return float(special.ndtri(self.quantile))  # == scipy.stats.norm.ppf

  def compute(self, truth) -> xl.Dataset:
    clim = xl.from_xarray(self.climatology)
    variables = [str(k) for k in truth.keys()]
    mean = _get_climatology_mean(clim, variables)
    std = _get_climatology_std(clim, variables)
    out = xl.Dataset()
    for name in variables:
      m = _materialise(mean[name], _selection_maps(mean[name], truth,
                                                   truth[name]))
      s = _materialise(std[name], _selection_maps(std[name], truth,
                                                  truth[name]))
      # np.float64 scalar * float32 array -> float64 (NumPy 2 promotion)
      thr = np.asarray(m.values) + np.float64(self.z()) * np.asarray(
          s.values, dtype=np.float64)
      out[name] = xl.DataArray(thr, m.dims, m.coords, name)
    return out

  def kernel_operands(self, truth, name, like, layout):
    clim = xl.from_xarray(self.climatology)
    mean = _get_climatology_mean(clim, [name])[name]
    std = _get_climatology_std(clim, [name])[name]
    m_op = sp.gather_operand(sp.prepare_operand(mean, layout, np.float32),
                             _selection_maps(mean, truth, like))
    s_op = sp.gather_operand(sp.prepare_operand(std, layout, np.float32),
                             _selection_maps(std, truth, like))
    return 'gaussian', m_op, s_op, self.z()


def get_threshold_cls(threshold_method: str) -> type:
  """thresholds.py:188-197."""
  if threshold_method == 'quantile':
    return QuantileThreshold
  if threshold_method == 'gaussian_quantile':
    return GaussianQuantileThreshold
  raise NotImplementedError(f'Unknown threshold method: {threshold_method}')

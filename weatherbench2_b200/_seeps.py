"""SEEPS / SpatialSEEPS -- same classes as weatherbench2/metrics.py:417-528 --
on top of K9 (csrc/seeps.cu) and, for the spatial mean, K1.

Imported into `weatherbench2_b200.metrics`; use them from there.
"""
from __future__ import annotations

import dataclasses
import functools
import typing as t

import numpy as np
import pandas as pd

from weatherbench2_b200 import _spatial as sp
from weatherbench2_b200 import metrics as m
from weatherbench2_b200 import xarray_lite as xl


def _valid_time(da: xl.DataArray):
  """(dims, timestamps) of `da.valid_time` (metrics.py:446-448); data indexed
  by valid time directly carry it as `time`."""
  for key in ('valid_time', 'time'):
    if key in da.coords:
      c = da.coords[key]
      return tuple(c.dims), np.asarray(c.values)
  raise AttributeError(f'{da.name!r} has no valid_time coordinate')


def _threshold_maps(wet_da: xl.DataArray, da: xl.DataArray) -> dict:
  """`.sel(dayofyear=valid_time.dt.dayofyear, hour=valid_time.dt.hour)` as
  index maps for the offset table (metrics.py:446-448)."""
  tdims, stamps = _valid_time(da)
  idx = pd.DatetimeIndex(stamps.ravel())
  maps = {}
  for dim, values in (('dayofyear', idx.dayofyear), ('hour', idx.hour)):
    if dim not in wet_da.dims:
      raise KeyError(f'{wet_da.name!r} has no {dim!r} dimension')
    pos = xl._lookup(wet_da.coords[dim].values, np.asarray(values))  # pylint: disable=protected-access
    maps[dim] = (tdims, pos.reshape(stamps.shape))
  return maps


@dataclasses.dataclass
class SpatialSEEPS(m.Metric):
  """Stable Equitable Error in Probability Space, per grid cell
  (metrics.py:417-513; Rodwell et al. 2010).

  Attributes as in the reference: `climatology` holds
  `<precip_name>_seeps_threshold` [m] and `<precip_name>_seeps_dry_fraction`.
  """

  climatology: t.Any = None
  dry_threshold_mm: float = 0.25
  precip_name: str = 'total_precipitation_24hr'
  min_p1: float = 0.1
  max_p1: float = 0.85

  def __hash__(self):
    return id(self)

  @functools.cached_property
  def p1(self) -> xl.DataArray:
    """Average dry fraction (metrics.py:441-444); a one-off host reduction of
    the climatology, like the latitude weights."""
    clim = xl.from_xarray(self.climatology)
    dry_fraction = clim[f'{self.precip_name}_seeps_dry_fraction']
    return dry_fraction.mean(('hour', 'dayofyear'))

  def _maps(self, forecast, truth, reduce_dim, skipna):
    ctx = m._context()  # pylint: disable=protected-access
    clim = xl.from_xarray(self.climatology)
    name = self.precip_name
    f_da, t_da = xl.align_inner(forecast[name], truth[name])
    wet_da = clim[f'{name}_seeps_threshold']
    for da in (f_da, t_da, wet_da):
      if da.dtype not in (np.float32, np.float64):
        raise TypeError(f'variable {da.name!r} has dtype {da.dtype}: SEEPS '
                        'takes float32 or float64 data')
    # each operand keeps its dtype: the kernel categorises in NumPy's
    # promoted precision, as the reference does (metrics.py:456-460)
    f_op = sp.prepare_operand(f_da, None)
    t_op = sp.prepare_operand(t_da, f_op.layout)
    w_op = sp.prepare_operand(wet_da, f_op.layout)
    maps, dims = sp.run_seeps_maps(
        ctx, f_op, t_op, w_op, _threshold_maps(wet_da, f_da),
        _threshold_maps(wet_da, t_da), self.p1, self.dry_threshold_mm / 1000.0,
        self.min_p1, self.max_p1, reduce_dim, skipna)
    out = xl.Dataset()
    out[name] = xl.DataArray(maps, dims, m._map_coords(dims, f_da, t_da), name)  # pylint: disable=protected-access
    return out

  def compute_chunk(self, forecast, truth, region=None, skipna=False):
    del region, skipna  # ignored (metrics.py:470): the p1 mask forces NaNs
    return self._maps(forecast, truth, None, False)

  def compute(self, forecast, truth, region=None, skipna=False):
    """metrics.py:117-138 with the time mean fused into the kernel."""
    del region
    return self._maps(forecast, truth, m._avg_dim(forecast), skipna)  # pylint: disable=protected-access


@dataclasses.dataclass
class SEEPS(SpatialSEEPS):
  """Spatially averaged SEEPS (metrics.py:516-528): the weighted mean of the
  maps with skipna = True (K1 on the device-resident maps)."""

  def __hash__(self):
    return id(self)

  def compute_chunk(self, forecast, truth, region=None, skipna=False):
    del skipna  # effectively True because of the p1 mask (metrics.py:526)
    out = self._maps(forecast, truth, None, False)
    return m._spatial_average(out, region=region, skipna=True)  # pylint: disable=protected-access

  def compute(self, forecast, truth, region=None, skipna=False):
    avg_dim = m._avg_dim(forecast)  # pylint: disable=protected-access
    return self.compute_chunk(forecast, truth, region=region,
                              skipna=skipna).mean(avg_dim, skipna=skipna)

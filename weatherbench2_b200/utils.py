"""Day-of-year climatologies (mean, standard deviation, quantiles and SEEPS
thresholds) on the GPU.

Drop-in for the climatology functions of weatherbench2/utils.py and the
computation of scripts/compute_climatology.py without Beam or zarr:

  create_window_weights      utils.py:73-85
  compute_hourly_stat        utils.py:143-166  (the `explicit` method)
  compute_daily_stat         utils.py:127-140
  compute_hourly_stat_fast   utils.py:217-272  (the `fast` method)
  compute_daily_stat_fast    utils.py:200-214, 275-287
  Quantile, SEEPSThreshold   compute_climatology.py:130-177
  compute_climatology        compute_climatology.py:219-356 (`main`)

The host turns the time selection into index tables (`_lib.ClimatologyPlan`):
the reference's year stacking over the union of day-of-year labels
(`xr.concat(dim='year')`, utils.py:97-103) or its `groupby('time.dayofyear')`.
The CUDA kernels read the (time, cells) series in place through them:
csrc/climatology.cu accumulates float64 moments and applies the circular
window (mean, std); csrc/climatology_quantile.cu slides a sorted window over
the day axis and takes xarray's weighted quantile of it (quantile, SEEPS).
CUDA tensors stay on the device; NumPy arrays (np.memmap included) are streamed
in bands of cells whose device footprint is bounded by `STREAM_BUDGET_BYTES`.

The quantile and SEEPS statistics exist for the `explicit` method only; the
`fast` functions refuse them, as the reference does.  `Quantile(qs).compute`
and `SEEPSThreshold(mm, var).compute` are accepted as `stat_fn` by
compute_hourly_stat / compute_daily_stat, which is how the reference script
passes them; calling `.compute` directly on other dimensions is not supported
(NotImplementedError).  At most 16 quantiles per call, and at most 8192
samples (stacked years x window_size) per window (ValueError).

Two deviations from the reference's compute_climatology: 'quantile' without
`quantiles=` raises NotImplementedError (the reference: ValueError), and
'seeps' without `seeps_dry_threshold_mm=` raises NotImplementedError instead
of defaulting to {'total_precipitation_24hr': 0.25,
'total_precipitation_6hr': 0.1}.  Statistics other than mean, std, quantile
and seeps are not computed (NotImplementedError).
"""
from __future__ import annotations

from typing import Callable, Optional, Sequence, Union

import numpy as np
import pandas as pd

from weatherbench2_b200 import _lib
from weatherbench2_b200 import _streamed
from weatherbench2_b200 import xarray_lite as xl

EXPLICIT, FAST = 0, 1
# device bytes of the two staging buffers of a NumPy input (one band of cells
# each: its selected time rows, resampled days and outputs)
STREAM_BUDGET_BYTES = 4 << 30

StatFn = Union[str, Callable[..., object]]


def create_window_weights(window_size: int) -> xl.DataArray:
  """Triangular weights over `window_size` days, normalised to mean 1."""
  assert window_size % 2 == 1, 'Window size must be odd.'
  half = window_size // 2
  w = np.concatenate([np.linspace(0, 1, half + 1),
                      np.linspace(1, 0, half + 1)[1:]])
  with np.errstate(invalid='ignore'):
    w = w / w.mean()
  return xl.DataArray(w, dims=['window'])


def _check_window(window_size: int):
  create_window_weights(window_size)  # AssertionError for an even size
  if window_size < 3:
    raise ValueError(f'window_size must be at least 3 (got {window_size}): '
                     'the triangular weights of a 1-day window are 0 / 0')


def _check_stat(stat_fn: StatFn, quantiles=None, seeps_dry_threshold_mm=None):
  if isinstance(stat_fn, str) and (
      stat_fn in ('mean', 'std') or
      (stat_fn == 'quantile' and quantiles is not None) or
      (stat_fn == 'seeps' and seeps_dry_threshold_mm is not None)):
    return
  hint = {'quantile': ' (pass quantiles=[...])',
          'seeps': ' (pass seeps_dry_threshold_mm={variable: mm})'}
  raise NotImplementedError(
      f'stat {stat_fn!r} not implemented: the GPU climatology computes the '
      "statistics 'mean' and 'std' (both methods), 'quantile' given quantiles= "
      "and 'seeps' given seeps_dry_threshold_mm= (explicit method); anything "
      'else is out of its scope' + hint.get(stat_fn, '')
      if isinstance(stat_fn, str) else
      f'stat {stat_fn!r} not implemented: only the explicit functions take '
      'Quantile(...).compute / SEEPSThreshold(...).compute; anything else is '
      'out of its scope')


class Quantile:
  """Weighted quantiles over (window, year) (compute_climatology.py:130-144).
  `stat_fn=Quantile(qs).compute` carries the quantiles into the GPU path."""

  def __init__(self, quantiles: Sequence[float]):
    self.quantiles = quantiles

  def compute(self, ds, dim, weights=None):
    raise NotImplementedError(
        'Quantile.compute runs inside compute_hourly_stat / compute_daily_stat '
        '(stat_fn=Quantile(qs).compute); other dimensions are out of its scope')


class SEEPSThreshold:
  """SEEPS heavy-precipitation threshold (the weighted 2/3 quantile of the wet
  samples) and dry fraction (compute_climatology.py:147-177).
  `stat_fn=SEEPSThreshold(mm, var).compute` carries them into the GPU path."""

  def __init__(self, dry_threshold_mm: float, var: str):
    self.dry_threshold_m = dry_threshold_mm / 1000.0
    self.var = var

  def compute(self, ds, dim, weights=None):
    raise NotImplementedError(
        'SEEPSThreshold.compute runs inside compute_hourly_stat / '
        'compute_daily_stat (stat_fn=SEEPSThreshold(mm, var).compute); other '
        'dimensions are out of its scope')


def _quantile_spec(stat_fn):
  """The Quantile / SEEPSThreshold a stat_fn carries, or None."""
  if isinstance(stat_fn, (Quantile, SEEPSThreshold)):
    return stat_fn
  owner = getattr(stat_fn, '__self__', None)
  if isinstance(owner, (Quantile, SEEPSThreshold)) and getattr(
      stat_fn, '__func__', None) is type(owner).compute:
    return owner
  return None


def _quantile_values(quantiles) -> np.ndarray:
  q = np.atleast_1d(np.asarray(quantiles, dtype=np.float64))
  if q.ndim != 1 or not q.size:
    raise ValueError(f'quantiles must be a non-empty sequence, got {quantiles!r}')
  if not np.all((q >= 0) & (q <= 1)):
    raise ValueError(f'Quantiles must be in the range [0, 1], got {quantiles!r}')
  if q.size > _lib.CLIM_MAX_QUANTILES:
    raise ValueError(f'at most {_lib.CLIM_MAX_QUANTILES} quantiles per call '
                     f'(got {q.size})')
  return q


# -- index tables -------------------------------------------------------------
def _select(times: pd.DatetimeIndex, clim_years) -> np.ndarray:
  """Indices of `obs.sel(time=clim_years)` (label slice, partial strings)."""
  if not isinstance(clim_years, slice):
    raise TypeError(f'clim_years must be a slice, got {clim_years!r}')
  start = None if clim_years.start is None else str(clim_years.start)
  stop = None if clim_years.stop is None else str(clim_years.stop)
  return np.arange(times.size)[times.slice_indexer(start, stop)]


def _explicit_slots(times: pd.DatetimeIndex, idx: np.ndarray):
  """Years stacked on the sorted union of their day-of-year labels; the fill
  source of every year is its day-365 step (utils.py:97-105)."""
  uy, yi = np.unique(np.asarray(times.year)[idx], return_inverse=True)
  ud, di = np.unique(np.asarray(times.dayofyear)[idx], return_inverse=True)
  if np.unique(di * uy.size + yi).size != idx.size:
    raise ValueError('more than one time step per year and day of year')
  items = np.full((ud.size, uy.size), -1, np.int64)
  items[di, yi] = idx
  pos = int(np.searchsorted(ud, 365))
  if pos == ud.size or ud[pos] != 365:
    raise KeyError(365)  # stacked.sel(dayofyear=365)
  return ud, items, items[pos].copy()


def _fast_slots(times: pd.DatetimeIndex, idx: np.ndarray):
  """groupby('time.dayofyear'): every step of a label feeds its slot."""
  ud, di = np.unique(np.asarray(times.dayofyear)[idx], return_inverse=True)
  counts = np.bincount(di, minlength=ud.size)
  order = np.argsort(di, kind='stable')
  rank = np.arange(idx.size) - np.repeat(np.cumsum(counts) - counts, counts)
  items = np.full((ud.size, int(counts.max())), -1, np.int64)
  items[di[order], rank] = idx[order]
  return ud, items, None


def _daily_resample(times: pd.DatetimeIndex, idx: np.ndarray):
  """resample(time='D'): every calendar day from the first to the last
  selected step; day i averages `count[i]` consecutive steps from `start[i]`."""
  ts = times[idx]
  if not ts.is_monotonic_increasing or np.any(np.diff(idx) != 1):
    raise ValueError('the daily resample needs a sorted time axis')
  day = ts.floor('D')
  days = pd.date_range(day[0], day[-1], freq='D')
  k = np.asarray((day - days[0]) // pd.Timedelta(days=1), dtype=np.int64)
  count = np.bincount(k, minlength=days.size).astype(np.int32)
  start = np.zeros(days.size, np.int64)
  start[k[::-1]] = idx[::-1]  # first step of each day
  return days, start, count


def _plan(times, clim_years, hours: Optional[Sequence[int]], method: int,
          resample: bool, window_size: int):
  """(ClimatologyPlan, day-of-year labels of the output)."""
  times = pd.DatetimeIndex(times)
  idx = _select(times, clim_years)
  res = (None, None)
  if resample:
    if not idx.size:
      raise ValueError(f'no time steps in {clim_years}')
    times, start, count = _daily_resample(times, idx)
    idx = np.arange(times.size)
    res = (start, count)
  slots = _explicit_slots if method == EXPLICIT else _fast_slots
  per_hour = []
  for hour in ([None] if hours is None else hours):
    sel = idx if hour is None else idx[np.asarray(times.hour)[idx] == hour]
    if not sel.size:  # the reference's xr.concat([]) / empty groupby
      raise ValueError(f'no time steps at hour {hour} in {clim_years}')
    per_hour.append(slots(times, sel))
  labels = np.unique(np.concatenate([p[0] for p in per_hour]))
  nhour = len(per_hour)
  nday = max(p[0].size for p in per_hour)
  nitem = max(p[1].shape[1] for p in per_hour)
  items = np.full((nhour, nday, nitem), -1, np.int64)
  fill = np.full((nhour, nitem), -1, np.int64)
  hour_nday = np.zeros(nhour, np.int32)
  out_row = np.zeros((nhour, nday), np.int32)
  for h, (ud, it, fl) in enumerate(per_hour):
    items[h, :ud.size, :it.shape[1]] = it
    if fl is not None:
      fill[h, :fl.size] = fl
    hour_nday[h] = ud.size
    out_row[h, :ud.size] = np.searchsorted(labels, ud)
  plan = _lib.ClimatologyPlan(items, fill if method == EXPLICIT else None,
                              hour_nday, out_row, labels.size, window_size,
                              method, *res)
  return plan, labels


# -- execution ------------------------------------------------------------------
def _series(da: xl.DataArray, plan):
  """(perm, dtype, other dims, their shape, ncell, ntime) of the (time, cells)
  series the kernels read: time first, float64 kept unless resampled, every
  other dtype read as float32."""
  ti = da.dims.index('time')
  other = tuple(d for d in da.dims if d != 'time')
  oshape = tuple(da.sizes[d] for d in other)
  ncell = int(np.prod(oshape)) if oshape else 1
  perm = [ti] + [i for i in range(len(da.dims)) if i != ti]
  # by name: a CUDA tensor may hold a dtype NumPy lacks (bfloat16)
  f64 = str(da.data.dtype).replace('torch.', '') == 'float64'
  dt = np.float64 if f64 and not plan.nres else np.float32
  return perm, dt, other, oshape, ncell, da.sizes['time']


def _run(ds: xl.Dataset, plan, labels, hours, stats: Sequence[str]) -> dict:
  """{stat: {variable: DataArray}} for every variable with a time axis."""
  out = {s: {} for s in stats}
  for name, da in ds.items():
    if 'time' not in da.dims:
      continue
    perm, dt, other, oshape, ncell, ntime = _series(da, plan)
    nrow = (plan.nhour, plan.nday_out)
    res = _streamed.run(
        'climatology', da.data, (ntime, ncell, plan),
        [(nrow + oshape, np.float32) if s in stats else None
         for s in ('mean', 'std')], STREAM_BUDGET_BYTES, perm=perm, dtype=dt)
    res = dict(zip(('mean', 'std'), res))
    res = {s: res[s] for s in stats}
    coords = {k: c for k, c in da.coords.items() if 'time' not in c.dims}
    coords['dayofyear'] = xl.Coord(('dayofyear',), labels)
    if hours is None:
      dims = ('dayofyear',) + other
      res = {s: v.reshape(nrow[1:] + oshape) for s, v in res.items()}
    else:
      dims = ('hour', 'dayofyear') + other
      coords['hour'] = xl.Coord(('hour',), np.asarray(hours))
    for s in stats:
      out[s][name] = xl.DataArray(res[s], dims, coords, name, da.attrs)
  return out


def _compute(ds, window_size: int, clim_years: slice,
             hours: Optional[Sequence[int]], method: int,
             stats: Sequence[str]) -> dict:
  """{stat: lite Dataset}; the daily fast mean averages the raw steps, every
  other daily statistic the daily resample (utils.py:200-214)."""
  _check_window(window_size)
  for s in stats:
    _check_stat(s)
  times = ds.coords['time'].values
  groups = [(list(stats), hours is None and method == EXPLICIT)]
  if hours is None and method == FAST:
    groups = [([s], s == 'std') for s in stats]
  out = {}
  for group, resample in groups:
    plan, labels = _plan(times, clim_years, hours, method, resample,
                         window_size)
    for s, variables in _run(ds, plan, labels, hours, group).items():
      out[s] = xl.Dataset(variables, attrs=ds.attrs)
  return out


def _run_quantile(ds: xl.Dataset, plan, labels, hours, spec) -> dict:
  """{name: DataArray}: the quantiles of every variable with a time axis
  (names kept), or the SEEPS pair of `spec.var`."""
  seeps = isinstance(spec, SEEPSThreshold)
  qs = np.array([2 / 3]) if seeps else _quantile_values(spec.quantiles)
  thr = spec.dry_threshold_m if seeps else None
  names = [spec.var] if seeps else [n for n, da in ds.items()
                                    if 'time' in da.dims]
  lead = ('dayofyear',) if hours is None else ('hour', 'dayofyear')
  out = {}
  for name in names:
    da = ds[name]
    perm, dt, other, oshape, ncell, ntime = _series(da, plan)
    qshape = (plan.nhour, qs.size, plan.nday_out) + oshape
    dshape = (plan.nhour, plan.nday_out) + oshape
    res, dry = _streamed.run(
        'climatology_quantile', da.data, (ntime, ncell, plan, qs, thr),
        [(qshape, np.float32), (dshape, np.float32) if seeps else None],
        STREAM_BUDGET_BYTES, perm=perm, dtype=dt)
    coords = {k: c for k, c in da.coords.items() if 'time' not in c.dims}
    coords['dayofyear'] = xl.Coord(('dayofyear',), labels)
    if hours is not None:
      coords['hour'] = xl.Coord(('hour',), np.asarray(hours))
    dims = lead + other
    shape = dshape[1:] if hours is None else dshape
    if seeps:
      for key, v in ((f'{name}_seeps_threshold', res.reshape(shape)),
                     (f'{name}_seeps_dry_fraction', dry.reshape(shape))):
        out[key] = xl.DataArray(v, dims, coords, key, da.attrs)
    else:
      coords['quantile'] = xl.Coord(('quantile',), qs)
      if hours is None:
        dims = ('quantile',) + dims
        v = res.reshape(qshape[1:])
      else:
        dims = ('hour', 'quantile') + dims[1:]
        v = res
      out[name] = xl.DataArray(v, dims, coords, name, da.attrs)
  return out


def _compute_quantile(ds, window_size: int, clim_years: slice,
                      hours: Optional[Sequence[int]], spec) -> xl.Dataset:
  """The Quantile / SEEPSThreshold climatology, explicit method; the daily
  statistics take the daily resample (utils.py:127-140)."""
  _check_window(window_size)
  if not isinstance(spec, SEEPSThreshold):
    _quantile_values(spec.quantiles)
  if isinstance(spec, SEEPSThreshold) and spec.var not in ds:
    raise KeyError(spec.var)
  plan, labels = _plan(ds.coords['time'].values, clim_years, hours, EXPLICIT,
                       hours is None, window_size)
  if plan.nitem * window_size > _lib.CLIM_QUANTILE_MAX_SAMPLES:
    raise ValueError(
        f'{plan.nitem} stacked years x window_size {window_size} exceeds the '
        f'{_lib.CLIM_QUANTILE_MAX_SAMPLES} samples per window of the GPU '
        'quantile climatology')
  return xl.Dataset(_run_quantile(ds, plan, labels, hours, spec),
                    attrs=ds.attrs)


def _hours(hour_interval: int):
  return list(range(0, 24, hour_interval))


@xl.boundary
def compute_hourly_stat(obs, window_size: int, clim_years: slice,
                        hour_interval: int, stat_fn: StatFn = 'mean'):
  """Climatology by hour of day and day of year, `explicit` method."""
  spec = _quantile_spec(stat_fn)
  if spec is not None:
    return _compute_quantile(obs, window_size, clim_years,
                             _hours(hour_interval), spec)
  _check_stat(stat_fn)
  res = _compute(obs, window_size, clim_years, _hours(hour_interval), EXPLICIT,
                 [stat_fn])
  return res[stat_fn]


@xl.boundary
def compute_daily_stat(obs, window_size: int, clim_years: slice,
                       stat_fn: StatFn = 'mean'):
  """Climatology by day of year of the daily means, `explicit` method."""
  spec = _quantile_spec(stat_fn)
  if spec is not None:
    return _compute_quantile(obs, window_size, clim_years, None, spec)
  _check_stat(stat_fn)
  res = _compute(obs, window_size, clim_years, None, EXPLICIT, [stat_fn])
  return res[stat_fn]


@xl.boundary
def compute_hourly_stat_fast(obs, window_size: int, clim_years: slice,
                             hour_interval: int, stat_fn: str = 'mean'):
  """Per-day mean / std by hour of day, smoothed over the window (`fast`)."""
  _check_stat(stat_fn)
  res = _compute(obs, window_size, clim_years, _hours(hour_interval), FAST,
                 [stat_fn])
  return res[stat_fn]


@xl.boundary
def compute_daily_stat_fast(obs, window_size: int, clim_years: slice,
                            stat_fn: str = 'mean'):
  """Per-day mean (raw steps) / std (daily means), smoothed (`fast`)."""
  _check_stat(stat_fn)
  res = _compute(obs, window_size, clim_years, None, FAST, [stat_fn])
  return res[stat_fn]


@xl.boundary
def compute_climatology(obs, *, frequency: str = 'hourly',
                        hour_interval: int = 1, window_size: int = 61,
                        start_year: int = 1990, end_year: int = 2020,
                        statistics: Sequence[str] = ('mean',),
                        method: str = 'explicit',
                        quantiles: Optional[Sequence[float]] = None,
                        seeps_dry_threshold_mm: Optional[dict] = None):
  """scripts/compute_climatology.py without Beam or zarr: variables without a
  time axis are dropped, time is selected over [start_year, end_year] (both
  inclusive), the mean keeps the variable's name, the std is `<var>_std` and
  the quantiles `<var>_quantile` (dims hour, quantile, dayofyear, ...).  SEEPS
  gives `<var>_seeps_threshold` and `<var>_seeps_dry_fraction` for the
  variables of `seeps_dry_threshold_mm` ({variable: dry threshold in mm}).
  Dims (hour, dayofyear, ...) for hourly, (dayofyear, ...) for daily; the day
  axis holds the day-of-year labels present in the selection.  Mean and std
  are computed from one read of the data."""
  stats = [statistics] if isinstance(statistics, str) else list(statistics)
  for s in stats:
    _check_stat(s, quantiles, seeps_dry_threshold_mm)
  if frequency not in ('hourly', 'daily'):
    raise NotImplementedError(f'Frequency {frequency} not implemented.')
  if method not in ('explicit', 'fast'):
    raise NotImplementedError(
        f'method {method} for climatological frequency {frequency} not '
        'implemented.')
  if method != 'explicit':
    if 'seeps' in stats:
      raise NotImplementedError('SEEPS only tested for explicit.')
    if 'quantile' in stats:
      raise NotImplementedError(f'stat {Quantile(quantiles).compute} not '
                                'implemented.')
  if 'quantile' in stats:
    _quantile_values(quantiles)
  hours = _hours(hour_interval) if frequency == 'hourly' else None
  years = slice(str(start_year), str(end_year))
  moments = [s for s in stats if s in ('mean', 'std')]
  res = (_compute(obs, window_size, years, hours,
                  EXPLICIT if method == 'explicit' else FAST, moments)
         if moments else {})
  out = xl.Dataset(attrs=obs.attrs)
  for s in stats:
    if s == 'quantile':
      q = _compute_quantile(obs, window_size, years, hours,
                            Quantile(quantiles))
      for name, da in q.items():
        da.name = f'{name}_quantile'
        out[da.name] = da
    elif s == 'seeps':
      for var, mm in seeps_dry_threshold_mm.items():
        for name, da in _compute_quantile(obs, window_size, years, hours,
                                          SEEPSThreshold(mm, var)).items():
          out[name] = da
    else:
      for name, da in res[s].items():
        key = name if s == 'mean' else f'{name}_{s}'
        da.name = key
        out[key] = da
  return out

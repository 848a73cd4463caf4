"""Float64 NumPy restatement of the reference's climatology computation
(weatherbench2/utils.py:38-44, 73-287; scripts/compute_climatology.py), step
by step and without shortcuts: stack the years on the union of their
day-of-year labels, fill from day 365, wrap-pad, weighted reduction over
(window, year); for the fast method, groupby day of year, then roll and
average.  The GPU operators of weatherbench2_b200.utils are checked against it.

Arrays have time on axis 0; `times` are datetime64 values.  Every function
returns (day-of-year labels, values) with values [hour][day][...] for the
hourly statistics and [day][...] for the daily ones.
"""
import numpy as np
import pandas as pd


def window_weights(window_size):
  """utils.create_window_weights (utils.py:73-85)."""
  assert window_size % 2 == 1, 'Window size must be odd.'
  half = window_size // 2
  w = np.concatenate([np.linspace(0, 1, half + 1),
                      np.linspace(1, 0, half + 1)[1:]])
  return w / w.mean()


def select_years(times, x, clim_years):
  """obs.sel(time=slice('Y0', 'Y1')): label slice with partial strings."""
  t = pd.DatetimeIndex(times)
  sl = t.slice_indexer(clim_years.start, clim_years.stop)
  return t[sl], x[sl]


def select_hour(times, x, hour):
  """utils.select_hour (utils.py:38-44): keep the hour, drop the time of day."""
  keep = np.asarray(times.hour == hour)
  return pd.DatetimeIndex(times[keep].floor('D')), x[keep]


def resample_daily(times, x):
  """resample(time='D').mean(): every calendar day from the first to the last
  step, NaN-skipping mean, NaN for a day without data."""
  day = times.floor('D')
  days = pd.date_range(day[0], day[-1], freq='D')
  out = np.full((days.size,) + x.shape[1:], np.nan)
  xd = x.astype(np.float64)
  for i, d in enumerate(days):
    sel = np.asarray(day == d)
    if sel.any():
      with np.errstate(invalid='ignore'), _quiet():
        out[i] = np.nanmean(xd[sel], axis=0)
  return days, out


def rolling_stat(times, x, window_size, stat):
  """utils.compute_rolling_stat (utils.py:88-124), explicit method."""
  w = window_weights(window_size)
  half = window_size // 2
  t = pd.DatetimeIndex(times)
  years = np.unique(t.year)
  if not years.size:
    raise ValueError('must supply at least one object to concatenate')
  labels = np.unique(t.dayofyear)  # the outer join of xr.concat(dim='year')
  stacked = np.full((years.size, labels.size) + x.shape[1:], np.nan)
  for yi, y in enumerate(years):
    sel = np.asarray(t.year == y)
    pos = np.searchsorted(labels, np.asarray(t.dayofyear[sel]))
    stacked[yi, pos] = x[sel]
  # stacked.fillna(stacked.sel(dayofyear=365)): per year, on any day
  if 365 not in labels:
    raise KeyError(365)
  fill = stacked[:, int(np.searchsorted(labels, 365))]
  stacked = np.where(np.isnan(stacked), fill[:, None], stacked)
  # pad(mode='wrap') then rolling(center=True).construct('window')
  pad = [(0, 0), (half, half)] + [(0, 0)] * (x.ndim - 1)
  padded = np.pad(stacked, pad, mode='wrap')
  out = np.full((labels.size,) + x.shape[1:], np.nan)
  for d in range(labels.size):
    out[d] = weighted_stat(padded[:, d:d + window_size], w, stat)
  return labels, out


def weighted_stat(win, w, stat):
  """xarray's weighted mean / population std of one window win (year, window,
  ...) over (year, window) with the tap weights w [window], NaN skipped; NaN
  where the weight sum is 0."""
  wb = np.asarray(w, np.float64).reshape((1, -1) + (1,) * (win.ndim - 2))
  ok = ~np.isnan(win)
  sw = (wb * ok).sum(axis=(0, 1))
  with np.errstate(invalid='ignore', divide='ignore'):
    mean = np.where(ok, wb * win, 0.0).sum(axis=(0, 1)) / sw
    if stat == 'mean':
      res = mean
    else:
      dev = np.where(ok, wb * (win - mean) ** 2, 0.0).sum(axis=(0, 1))
      res = np.sqrt(dev / sw)
  return np.where(sw == 0, np.nan, res)


def dayofyear_stat(times, x, stat):
  """groupby('time.dayofyear').mean() / .std() (ddof 0, NaN skipped)."""
  t = pd.DatetimeIndex(times)
  labels = np.unique(t.dayofyear)
  if not labels.size:
    raise ValueError('empty groupby')
  out = np.full((labels.size,) + x.shape[1:], np.nan)
  for i, d in enumerate(labels):
    v = x[np.asarray(t.dayofyear == d)].astype(np.float64)
    with np.errstate(invalid='ignore'), _quiet():
      out[i] = np.nanmean(v, axis=0) if stat == 'mean' else np.nanstd(v, axis=0)
  return labels, out


def smooth_dayofyear(values, window_size):
  """utils.smooth_dayofyear_variable_with_rolling_window (utils.py:169-197):
  mean over i of w[i] * roll(values, i), NaN skipped (count denominator)."""
  w = window_weights(window_size)
  half = window_size // 2
  stack = np.stack([np.roll(values, i, axis=0) * w[i + half]
                    for i in np.arange(-half, window_size - half)])
  with _quiet():
    return np.nanmean(stack, axis=0)


def _concat_hours(per_hour):
  """xr.concat over hours: outer join of the day labels, NaN where missing."""
  labels = np.unique(np.concatenate([p[0] for p in per_hour]))
  shape = per_hour[0][1].shape[1:]
  out = np.full((len(per_hour), labels.size) + shape, np.nan)
  for h, (lab, v) in enumerate(per_hour):
    out[h, np.searchsorted(labels, lab)] = v
  return labels, out


def hourly_stat(times, x, window_size, clim_years, hour_interval, stat):
  """utils.compute_hourly_stat (utils.py:143-166)."""
  t, v = select_years(times, x, clim_years)
  return _concat_hours([
      rolling_stat(*select_hour(t, v, hour), window_size, stat)
      for hour in range(0, 24, hour_interval)])


def daily_stat(times, x, window_size, clim_years, stat):
  """utils.compute_daily_stat (utils.py:127-140)."""
  t, v = select_years(times, x, clim_years)
  return rolling_stat(*resample_daily(t, v), window_size, stat)


def hourly_stat_fast(times, x, window_size, clim_years, hour_interval, stat):
  """utils.compute_hourly_stat_fast (utils.py:217-272)."""
  t, v = select_years(times, x, clim_years)
  per_hour = []
  for hour in range(0, 24, hour_interval):
    labels, vals = dayofyear_stat(*select_hour(t, v, hour), stat)
    per_hour.append((labels, smooth_dayofyear(vals, window_size)))
  return _concat_hours(per_hour)


def daily_stat_fast(times, x, window_size, clim_years, stat):
  """utils.compute_daily_stat_fast (utils.py:200-214, 275-287): the mean
  groups the raw steps, the std the daily means."""
  t, v = select_years(times, x, clim_years)
  if stat == 'std':
    t, v = resample_daily(t, v)
  labels, vals = dayofyear_stat(t, v, stat)
  return labels, smooth_dayofyear(vals, window_size)


class _quiet:
  def __enter__(self):
    import warnings  # pylint: disable=import-outside-toplevel
    self._cm = warnings.catch_warnings()
    self._cm.__enter__()
    warnings.simplefilter('ignore', RuntimeWarning)

  def __exit__(self, *exc):
    return self._cm.__exit__(*exc)

"""Float64 NumPy restatement of the reference's quantile and SEEPS
climatologies (scripts/compute_climatology.py:130-177 called from
weatherbench2/utils.py:88-166, the explicit method), step by step: stack the
years on the union of their day-of-year labels, fill from day 365, wrap-pad,
construct the window, then xarray's weighted type-7 quantile of every
(day, cell) window literally (skipna, zero weights dropped, Kish's effective
size, sorted cumulative weights).

Arrays have time on axis 0; `times` are datetime64 values.  Every function
returns (day-of-year labels, values): quantiles [hour][quantile][day][...]
(hourly) or [quantile][day][...] (daily); SEEPS (threshold, dry fraction)
each [hour][day][...] or [day][...].
"""
import numpy as np
import pandas as pd

import climatology_oracle as co


def weighted_quantile(data, weights, quantiles):
  """xarray's weighted quantile of one sample set (Akinshin's type 7)."""
  data = np.asarray(data, np.float64).ravel()
  weights = np.asarray(weights, np.float64).ravel()
  q = np.atleast_1d(np.asarray(quantiles, np.float64))
  keep = ~np.isnan(data)  # skipna
  data, weights = data[keep], weights[keep]
  keep = weights != 0
  data, weights = data[keep], weights[keep]
  if not data.size:
    return np.full(q.size, np.nan)
  nw = weights.sum() ** 2 / (weights ** 2).sum()
  order = np.argsort(data, kind='stable')
  data, weights = data[order], weights[order]
  weights = weights / weights.sum()
  c = np.append(0.0, np.cumsum(weights))
  h = np.clip((nw - 1) * q[:, None] + 1, 1, nw)
  u = np.maximum((h - 1) / nw, np.minimum(h / nw, c))
  v = u * nw - h + 1
  return (data * np.diff(v, axis=1)).sum(axis=1)


def seeps_of_window(samples, weights, dry_threshold):
  """SEEPSThreshold.compute of one window: (the weighted 2/3 quantile of the
  samples that are not dry, the unweighted fraction of dry samples)."""
  samples = np.asarray(samples)
  dry = samples < dry_threshold
  wet = np.where(dry, np.nan, samples)
  return [weighted_quantile(wet, weights, 2 / 3)[0], dry.mean()]


def rolling_windows(times, x, window_size):
  """compute_rolling_stat up to the reduction: (labels, [day][year][window]
  [...]) in x's dtype."""
  half = window_size // 2
  t = pd.DatetimeIndex(times)
  years = np.unique(t.year)
  if not years.size:
    raise ValueError('must supply at least one object to concatenate')
  labels = np.unique(t.dayofyear)
  stacked = np.full((years.size, labels.size) + x.shape[1:], np.nan, x.dtype)
  for yi, y in enumerate(years):
    sel = np.asarray(t.year == y)
    stacked[yi, np.searchsorted(labels, np.asarray(t.dayofyear[sel]))] = x[sel]
  if 365 not in labels:
    raise KeyError(365)
  fill = stacked[:, int(np.searchsorted(labels, 365))]
  stacked = np.where(np.isnan(stacked), fill[:, None], stacked)
  pad = [(0, 0), (half, half)] + [(0, 0)] * (x.ndim - 1)
  padded = np.pad(stacked, pad, mode='wrap')
  win = np.stack([padded[:, d:d + window_size] for d in range(labels.size)])
  return labels, win


def _per_cell(win, weights, fn):
  """fn(samples, weights) for every (day, cell) of [day][year][window][...]."""
  wts = np.broadcast_to(weights, win.shape[1:3])
  out = None
  for d in range(win.shape[0]):
    for cell in np.ndindex(win.shape[3:]):
      r = np.asarray(fn(win[(d, slice(None), slice(None)) + cell], wts))
      if out is None:
        out = np.full((win.shape[0],) + win.shape[3:] + r.shape, np.nan)
      out[(d,) + cell] = r
  return np.moveaxis(out, -1, 0)  # [result][day][...]


def rolling_quantile(times, x, window_size, quantiles):
  """Quantile.compute on the rolling windows: [quantile][day][...]."""
  labels, win = rolling_windows(times, x, window_size)
  w = co.window_weights(window_size)
  return labels, _per_cell(win, w, lambda s, ws: weighted_quantile(
      s, ws, quantiles))


def rolling_seeps(times, x, window_size, dry_threshold_m):
  """SEEPSThreshold.compute on the rolling windows: the comparison runs in
  x's precision (NumPy 2 rounds the Python float to it); the dry fraction is
  the unweighted mean over (year, window), NaN never dry."""
  labels, win = rolling_windows(times, x, window_size)
  w = co.window_weights(window_size)
  thr = x.dtype.type(dry_threshold_m)
  res = _per_cell(win, w, lambda s, ws: seeps_of_window(s, ws, thr))
  return labels, res[0], res[1]


def _series(times, x, clim_years, daily):
  t, v = co.select_years(times, x, clim_years)
  if daily:  # the daily means in float32, the precision the GPU reads
    t, v = co.resample_daily(pd.DatetimeIndex(t), v)
    v = v.astype(np.float32)
  return t, v


def hourly_quantile(times, x, window_size, clim_years, hour_interval,
                    quantiles):
  """compute_hourly_stat(stat_fn=Quantile(quantiles).compute)."""
  t, v = _series(times, x, clim_years, False)
  per_hour = []
  for hour in range(0, 24, hour_interval):
    labels, q = rolling_quantile(*co.select_hour(t, v, hour), window_size,
                                 quantiles)
    per_hour.append((labels, np.moveaxis(q, 0, 1)))
  labels, out = co._concat_hours(per_hour)  # pylint: disable=protected-access
  return labels, np.moveaxis(out, 2, 1)


def daily_quantile(times, x, window_size, clim_years, quantiles):
  """compute_daily_stat(stat_fn=Quantile(quantiles).compute)."""
  return rolling_quantile(*_series(times, x, clim_years, True), window_size,
                          quantiles)


def hourly_seeps(times, x, window_size, clim_years, hour_interval,
                 dry_threshold_mm):
  """compute_hourly_stat(stat_fn=SEEPSThreshold(mm, var).compute)."""
  t, v = _series(times, x, clim_years, False)
  thr, frac = [], []
  for hour in range(0, 24, hour_interval):
    labels, a, b = rolling_seeps(*co.select_hour(t, v, hour), window_size,
                                 dry_threshold_mm / 1000.0)
    thr.append((labels, a))
    frac.append((labels, b))
  labels, a = co._concat_hours(thr)  # pylint: disable=protected-access
  _, b = co._concat_hours(frac)  # pylint: disable=protected-access
  return labels, a, b


def daily_seeps(times, x, window_size, clim_years, dry_threshold_mm):
  """compute_daily_stat(stat_fn=SEEPSThreshold(mm, var).compute)."""
  return rolling_seeps(*_series(times, x, clim_years, True), window_size,
                       dry_threshold_mm / 1000.0)

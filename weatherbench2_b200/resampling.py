"""Resampling and rolling windows in time on the GPU: mean, min, max and sum.

Drop-in for scripts/resample_in_time.py without Beam or zarr:

  resample_in_time_core   resample_in_time.py:270-309 (TIME_DIM and LABEL_SIDE
                          are keyword arguments here)
  resample_in_time        resample_in_time.py:312-451 (`main`)

Datasets may be xarray or xarray_lite; the result is of the same kind.  Data
may be NumPy (np.memmap included) or CUDA tensors; CUDA input gives CUDA
output.  The series is read in place as [outer][time][inner] by
csrc/resample.cu, and every statistic asked of a variable comes from one read
of it (the reference makes one pass per statistic).  NumPy input is streamed
in bands whose device footprint is bounded by `STREAM_BUDGET_BYTES`.

The bins of `resample` come from pandas: the positions 0..n-1 grouped by
`pd.Series(positions, index=times).resample(period, label=..., closed=...)`,
the grouper xarray delegates to, so labels and bin edges match it for
DatetimeIndex and TimedeltaIndex axes.  Semantics of the statistics (NaN,
empty bins, Inf) are those of include/wb2b200.h and DESIGN.md section 8c.

Deviations from the reference: data must be float32 or float64 (TypeError
naming the variable; the output keeps the input's dtype); an empty bin gives
NaN for the sum too (xarray without flox); a statistic other than mean, min,
max and sum raises ValueError; variables without the time dimension pass
through resample_in_time_core unchanged.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np
import pandas as pd

from weatherbench2_b200 import _streamed
from weatherbench2_b200 import xarray_lite as xl

STATISTICS = ('mean', 'min', 'max', 'sum')
# device bytes of the two staging buffers of a NumPy input (one band each:
# its time series and outputs)
STREAM_BUDGET_BYTES = 4 << 30
_ALL = 'ALL'


def _bins(times, period: pd.Timedelta, label_side: str):
  """(labels, bin_start, bin_count) of resample(period) over a sorted axis:
  bin b holds the positions [bin_start[b], bin_start[b] + bin_count[b])."""
  index = pd.Index(times)
  if not index.is_monotonic_increasing:
    raise ValueError('index must be monotonic increasing for resampling')
  positions = pd.Series(np.arange(index.size), index=index)
  if label_side == 'left':
    grouped = positions.resample(period, label='left')
  elif label_side == 'right':
    grouped = positions.resample(period, label='right', closed='right')
  else:
    raise ValueError(f'Unhandled label_side={label_side!r}')
  counts = grouped.count()
  count = counts.to_numpy(np.int64)
  start = np.cumsum(count) - count  # the bins partition the sorted axis
  labels = counts.index.values
  if label_side == 'right':  # the reference's isel(slice(1, None))
    labels, start, count = labels[1:], start[1:], count[1:]
  return labels, start.astype(np.int64), count.astype(np.int32)


def _window(times, period: pd.Timedelta) -> int:
  """Steps per rolling window; `period` must be a multiple of the spacing of
  the first two times."""
  delta_t = pd.to_timedelta(np.diff(np.asarray(times)[:2])[0])
  if period % delta_t:
    raise ValueError(
        f'delta_t={delta_t!r} between chunk times did not evenly divide '
        f'period={period!r}')
  window = int(period // delta_t)
  if window < 1:
    raise ValueError(f'period={period!r} and delta_t={delta_t!r} give a window '
                     f'of {window} steps')
  return window


def _stats(da: xl.DataArray, time_dim: str, stats: Sequence[str],
           skipna: bool, bins=None, window: int = 0) -> dict:
  """{statistic: array} of one variable along `time_dim`, all statistics from
  one read; each array has the input's dims and dtype, `time_dim` resized."""
  if da.dtype not in (np.float32, np.float64):
    raise TypeError(f'variable {da.name!r} has dtype {da.dtype}: time '
                    'resampling takes float32 or float64 data')
  ti = da.dims.index(time_dim)
  shape = da.shape
  nouter = int(np.prod(shape[:ti], dtype=np.int64))
  ntime = shape[ti]
  ninner = int(np.prod(shape[ti + 1:], dtype=np.int64))
  start, count = bins if bins is not None else (None, None)
  nout = ntime if window else len(count)
  oshape = shape[:ti] + (nout,) + shape[ti + 1:]
  res = _streamed.run(
      'time_window_stats', da.data,
      (nouter, ntime, ninner, start, count, window, skipna),
      [(oshape, da.dtype) if s in stats else None for s in STATISTICS],
      STREAM_BUDGET_BYTES)
  res = dict(zip(STATISTICS, res))
  return {s: res[s] for s in stats}


def _plan(times, method: str, period: pd.Timedelta, label_side: str):
  """(output times, bins or None, window or 0) of one method."""
  if method == 'rolling':
    return np.asarray(times), None, _window(times, period)
  if method == 'resample':
    labels, start, count = _bins(times, period, label_side)
    return labels, (start, count), 0
  raise ValueError(f'Unhandled method={method!r}')


def _coords(ds, time_dim: str, times, method: str) -> dict:
  """The coordinates of the output: those without `time_dim`, the new time
  coordinate, and (rolling only) the others along `time_dim`."""
  out = {}
  for k, c in ds.coords.items():
    if time_dim not in c.dims or (method == 'rolling' and k != time_dim):
      out[k] = c
  old = ds.coords.get(time_dim)
  out[time_dim] = xl.Coord((time_dim,), times, old.attrs if old else None)
  return out


@xl.boundary
def resample_in_time_core(chunk, method: str, period, statistic: str,
                          skipna: bool, *, time_dim: str = 'time',
                          label_side: str = 'left'):
  """xarray's resample / rolling (min_periods=None) `statistic` along
  `time_dim`.  Resample windows are [T, T + period) labelled T (left) or
  (T - period, T] labelled T without the first bin (right); rolling output T
  reduces the `period // delta_t` steps ending at T."""
  period = pd.to_timedelta(period)
  if time_dim not in chunk.coords:
    raise KeyError(time_dim)
  times, bins, window = _plan(chunk.coords[time_dim].values, method, period,
                              label_side)
  if statistic not in STATISTICS:
    raise ValueError(f'Unhandled statistic={statistic!r}: one of {STATISTICS}')
  coords = _coords(chunk, time_dim, times, method)
  if isinstance(chunk, xl.DataArray):
    if time_dim not in chunk.dims:
      return chunk
    v = _stats(chunk, time_dim, [statistic], skipna, bins, window)[statistic]
    coords = {k: c for k, c in coords.items()
              if all(d in chunk.dims for d in c.dims)}
    return xl.DataArray(v, chunk.dims, coords, chunk.name, chunk.attrs)
  out = xl.Dataset(coords=coords, attrs=chunk.attrs)
  for name, da in chunk.items():
    if time_dim in da.dims:
      v = _stats(da, time_dim, [statistic], skipna, bins, window)[statistic]
      out[name] = xl.DataArray(v, da.dims, name=name, attrs=da.attrs)
    else:
      out[name] = da
  return out


def _get_vars(list_of_vars, time_dependent_vars) -> list:
  """The variables of one statistic: ['ALL'] is every time dependent one."""
  if isinstance(list_of_vars, str):
    list_of_vars = [list_of_vars]
  list_of_vars = list(list_of_vars or [])
  if not list_of_vars:
    return []
  if len(list_of_vars) == 1 and list_of_vars[0] == _ALL:
    return list(time_dependent_vars)
  if _ALL in list_of_vars:
    raise ValueError(
        f'Cannot specify both {_ALL} and other variables. Found {list_of_vars}')
  return list_of_vars


@xl.boundary
def resample_in_time(ds, *, period, method: str = 'resample',
                     mean_vars: Sequence[str] = (),
                     min_vars: Sequence[str] = (),
                     max_vars: Sequence[str] = (),
                     sum_vars: Sequence[str] = (), label_side: str = 'left',
                     add_mean_suffix: bool = False, skipna: bool = False,
                     time_dim: str = 'time', time_start: Optional[str] = None,
                     time_stop: Optional[str] = None):
  """scripts/resample_in_time.py without Beam or zarr.  Selects
  [time_start, time_stop] on `time_dim` (labels, both ends inclusive; partial
  date strings and Timedelta strings such as '9 days'), then gives `<var>`
  (or `<var>_mean` with add_mean_suffix), `<var>_min`, `<var>_max` and
  `<var>_sum` of the variables listed for each statistic ('ALL': every
  variable with `time_dim`).  Rolling labels output T with the window
  [T, T + period) (left) or (T - period, T] (right), so resample and rolling
  agree at common times.  All statistics of a variable come from one read."""
  period = pd.to_timedelta(period)
  if time_start is not None or time_stop is not None:
    index = pd.Index(ds.coords[time_dim].values)
    ds = ds.isel({time_dim: index.slice_indexer(time_start, time_stop)})
  time_vars = [k for k, v in ds.items() if time_dim in v.dims]
  wanted = {s: _get_vars(v, time_vars) for s, v in (
      ('mean', mean_vars), ('min', min_vars), ('max', max_vars),
      ('sum', sum_vars))}
  keep = set().union(*wanted.values())
  nontime = keep.intersection(set(ds).difference(time_vars))
  if nontime:
    raise ValueError('Statistics asked for on some variables that did not '
                     f'contain {time_dim}: {nontime}')
  missing = keep.difference(ds.keys())
  if missing:
    raise KeyError(f'variables not in the dataset: {sorted(missing)}')
  times = ds.coords[time_dim].values
  if method == 'rolling':
    delta_ts = pd.to_timedelta(np.unique(np.diff(times)))
    if len(delta_ts) != 1:
      raise ValueError(f'Input data must have constant spacing. Found {delta_ts}')
    delta_t = delta_ts[0]
    if label_side == 'left':
      times = times - period + delta_t
    elif label_side == 'right':
      times = times + delta_t
    else:
      raise ValueError(f'Unhandled label_side={label_side!r}')
  out_times, bins, window = _plan(times, method, period, label_side)
  per_var = {}
  for name in sorted(keep, key=time_vars.index):
    stats = [s for s in STATISTICS if name in wanted[s]]
    per_var[name] = _stats(ds[name], time_dim, stats, skipna, bins, window)
  out = xl.Dataset(coords=_coords(ds, time_dim, out_times, method),
                   attrs=ds.attrs)
  for s in STATISTICS:
    for name in wanted[s]:
      key = name if s == 'mean' and not add_mean_suffix else f'{name}_{s}'
      da = ds[name]
      out[key] = xl.DataArray(per_var[name][s], da.dims, name=key,
                              attrs=da.attrs)
  return out

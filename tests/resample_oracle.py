"""TEST INFRASTRUCTURE: float64 NumPy oracle of time resampling and rolling
windows, bin by bin and window by window, following the semantics table of
DESIGN.md section 8c (include/wb2b200.h, wb2_time_window_stats):

  resample, skipna False   any NaN in the bin -> NaN
  resample, skipna True    NaN skipped; all-NaN non-empty bin: mean / min / max
                           NaN, sum 0 (nansum)
  empty bin                NaN for every statistic, sum included
  rolling (window w)       output t reduces [t-w+1, t]; NaN when t < w-1 or
                           when any value of the window is NaN, whatever skipna
  +-Inf                    what NumPy float64 gives for the window
"""
import warnings

import numpy as np

STATISTICS = ('mean', 'min', 'max', 'sum')


def reduce(v: np.ndarray, statistic: str, skipna: bool) -> np.ndarray:
  """`statistic` over axis 0 of the float64 window `v` (n, ...)."""
  if v.shape[0] == 0:
    return np.full(v.shape[1:], np.nan)
  fns = ({'mean': np.nanmean, 'min': np.nanmin, 'max': np.nanmax,
          'sum': np.nansum} if skipna else
         {'mean': np.mean, 'min': np.min, 'max': np.max, 'sum': np.sum})
  with warnings.catch_warnings():
    warnings.simplefilter('ignore', RuntimeWarning)
    with np.errstate(invalid='ignore', over='ignore'):
      return fns[statistic](v, axis=0)


def resample(x, start, count, statistics=STATISTICS, skipna=False, axis=0):
  """{statistic: array}: output b reduces the count[b] steps from start[b]
  along `axis` of x (float64, the axis resized to the number of bins)."""
  xt = np.moveaxis(np.asarray(x, dtype=np.float64), axis, 0)
  out = {}
  for s in statistics:
    r = np.stack([reduce(xt[int(b0):int(b0) + int(c)], s, skipna)
                  for b0, c in zip(start, count)]) if len(count) else (
                      np.zeros((0,) + xt.shape[1:]))
    out[s] = np.moveaxis(r, 0, axis)
  return out


def rolling(x, window: int, statistics=STATISTICS, axis=0):
  """{statistic: array}: output t reduces steps [t-w+1, t] along `axis`; NaN
  before a full window and for any window holding a NaN."""
  xt = np.moveaxis(np.asarray(x, dtype=np.float64), axis, 0)
  out = {}
  for s in statistics:
    r = np.full(xt.shape, np.nan)
    for t in range(window - 1, xt.shape[0]):
      r[t] = reduce(xt[t - window + 1:t + 1], s, skipna=False)
    out[s] = np.moveaxis(r, 0, axis)
  return out

"""TEST ORACLE: the three reindexing operations restated label by label in
NumPy, independent of the offset tables of weatherbench2_b200.reindexing.
Each output element is found by looking its labels up in the source's
coordinates one at a time; NaN where the lookup finds nothing."""
import numpy as np
import pandas as pd


def _find(values, label):
  hits = np.flatnonzero(np.asarray(values) == label)
  return int(hits[0]) if hits.size else None


def expand_climatology(x, dims, dayofyear, hours, times):
  """x (dims incl. dayofyear[, hour]) -> (time, *others) by label."""
  times = pd.DatetimeIndex(times)
  others = [d for d in dims if d not in ('dayofyear', 'hour')]
  xt = np.moveaxis(x, [dims.index(d) for d in others],
                   list(range(len(x.shape) - len(others), len(x.shape))))
  lead = [d for d in dims if d in ('dayofyear', 'hour')]
  out = []
  for t in times:
    idx = []
    for d in lead:
      label = t.dayofyear if d == 'dayofyear' else t.hour
      i = _find(dayofyear if d == 'dayofyear' else hours, label)
      if i is None:
        raise KeyError(label)
      idx.append(i)
    out.append(xt[tuple(idx)])
  return np.stack(out), ('time',) + tuple(others)


def index_on_valid_time(x, dims, init, leads, offset, spacing, mode):
  """x (..., time, ..., prediction_timedelta, ...) on valid time, float32."""
  it, il = dims.index('time'), dims.index('prediction_timedelta')
  xt = np.moveaxis(x.astype(np.float64), [it, il], [0, 1])
  if mode == 'valid_and_delta':
    kept = np.arange(offset, len(leads), spacing)
    times = np.unique(init[:, None] + leads[kept][None, :])
    out = np.full((times.size, kept.size) + xt.shape[2:], np.nan)
    for a, t in enumerate(times):
      for b, k in enumerate(kept):
        i = _find(init, t - leads[k])
        if i is not None:
          out[a, b] = xt[i, k]
    odims = list(dims)
  else:
    times = np.unique(init[:, None] + leads[None, :])
    out = np.full((init.size, times.size) + xt.shape[2:], np.nan)
    for a in range(init.size):
      for b, t in enumerate(times):
        k = _find(leads, t - init[a])
        if k is not None:
          out[a, b] = xt[a, k]
    odims = ['init' if d == 'time' else 'time' if d == 'prediction_timedelta'
             else d for d in dims]
  out = np.moveaxis(out, [0, 1], [it, il]).astype(np.float32)
  return out, tuple(odims), times


def sample_forecasts(x, dims, truth_times, sampled, timedeltas,
                     time_dim='time'):
  """out[m, d, j] = x at time sampled[m, j] + timedeltas[d] (by label)."""
  it = dims.index(time_dim)
  xt = np.moveaxis(x, it, 0)
  sampled = np.asarray(sampled, 'datetime64[ns]')
  deltas = np.asarray(pd.TimedeltaIndex(timedeltas).values)
  out = np.empty(sampled.shape[:1] + deltas.shape + sampled.shape[1:] +
                 xt.shape[1:], x.dtype)
  for m in range(sampled.shape[0]):
    for d in range(deltas.size):
      for j in range(sampled.shape[1]):
        i = _find(truth_times, sampled[m, j] + deltas[d])
        if i is None:
          raise ValueError('missing time')
        out[m, d, j] = xt[i]
  return out, ('realization', 'prediction_timedelta', time_dim) + tuple(
      d for d in dims if d != time_dim)

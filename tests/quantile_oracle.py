"""NumPy oracle of wb2_quantile / wb2_quantile_host (include/wb2b200.h, DESIGN.md
section 8f): per cell numpy's np.quantile (skipna False) or np.nanquantile
(skipna True) with method 'linear' and float64 q, which is what xarray's
Dataset.quantile calls, cast to float64 (the entries' output type).

`contract` restates the header's six steps independently of numpy, so that
tests/test_quantile_cpu.py can tie the header's recipe to numpy bit for bit.
"""
import warnings

import numpy as np


def quantile(x, quantiles, skipna=False, axis=1):
  """np.quantile / np.nanquantile of `x` along `axis`, float64 out, with the
  quantile axis first (the entries' [nquantile][outer][inner] layout for a
  [outer][n][inner] series)."""
  q = np.asarray(quantiles, dtype=np.float64)
  fn = np.nanquantile if skipna else np.quantile
  with warnings.catch_warnings():
    warnings.simplefilter('ignore', RuntimeWarning)  # all-NaN slices
    res = fn(x, q, axis=axis, method='linear')
  return np.asarray(res, dtype=np.float64)


def contract(cell, quantiles, skipna=False):
  """The six steps of include/wb2b200.h for one cell of float32 / float64
  samples, in plain Python float arithmetic (each operation one correctly
  rounded double operation) and NumPy scalars for the T-rounded difference."""
  t = cell.dtype.type
  cell = np.asarray(cell)
  nan = np.isnan(cell)
  out = []
  for q in quantiles:
    q = float(q)
    if (nan.any() and not skipna) or nan.all():
      out.append(float('nan'))
      continue
    s = np.sort(cell[~nan])
    m = s.size
    v = float(m - 1) * q
    if v >= m - 1:
      i = j = m - 1
      g = v + 1.0
    else:
      i = int(np.floor(v))
      j = i + 1
      g = v - float(i)
    with np.errstate(invalid='ignore', over='ignore'):
      d = float(t(s[j]) - t(s[i]))
    a, b = float(s[i]), float(s[j])
    out.append(a + d * g if g < 0.5 else b - d * (1.0 - g))
  return np.asarray(out, dtype=np.float64)

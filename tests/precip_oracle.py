"""NumPy oracle of wb2_precip_accumulation (include/wb2b200.h, DESIGN.md
section 8e), restating PrecipitationAccumulation.compute
(weatherbench2/derived_variables.py:471-528) with the package's numerics:

  d[k]   = np.diff(x) in the data's dtype (xarray's diff)
  s      = d[t-w+1] + ... + d[t], an explicit float64 loop, oldest first
  out[t] = T(s); with clamp, T(s) < 0 -> +0.0 (NaN and -0.0 kept)
  out[t] = NaN for t < w

The reference sums float32 differences in float32; the gap to it is bounded
by `reference_bound`."""
import numpy as np


def accumulate(x, window: int, clamp: bool = True, axis: int = -1):
  """The accumulation of cumulative series `x` along `axis`; x's dtype."""
  x = np.asarray(x)
  dt = x.dtype
  xm = np.moveaxis(x, axis, -1)
  n = xm.shape[-1]
  out = np.full(xm.shape, np.nan, dt)
  if window < n:
    with np.errstate(invalid='ignore', over='ignore'):
      d = np.diff(xm, axis=-1)  # d[k-1] = x[k] - x[k-1], rounded in dt
      for t in range(window, n):
        s = d[..., t - window].astype(np.float64)
        for k in range(t - window + 1, t):
          s = s + d[..., k].astype(np.float64)
        r = s.astype(dt)
        if clamp:
          r = np.where(r < 0, dt.type(0), r)
        out[..., t] = r
  return np.moveaxis(out, -1, axis)


def reference_bound(x, window: int, axis: int = -1):
  """(w + 1) * 2^-24 * sum |d[k]| over each window: how far the float64
  accumulation of float32 differences may be from a float32 one."""
  xm = np.moveaxis(np.asarray(x, np.float64), axis, -1)
  n = xm.shape[-1]
  out = np.full(xm.shape, np.nan)
  d = np.abs(np.diff(xm, axis=-1))
  for t in range(window, n):
    out[..., t] = (window + 1) * 2.0**-24 * d[..., t - window:t].sum(-1)
  return np.moveaxis(out, -1, axis)

"""The column-integral contract of include/wb2b200.h (wb2_column_integral) in
NumPy: total column water, integrated water transport and eddy kinetic energy
of weatherbench2/derived_variables.py:212-228 and 365-430.  It does not import
the package.

Every function takes arrays with the level axis at `level_axis` and returns
the float64 value before the one rounding to the data type; `rounded` does
that rounding."""
import warnings

import numpy as np
import pandas as pd

INV_G = 1 / 9.81
EPS32 = 2.0 ** -24


def weights(level) -> np.ndarray:
  """w_k = 0.5 * (level[k+1] - level[k]), the level coordinate as float64."""
  return np.diff(np.asarray(level, np.float64)) * 0.5


def level_sum(y, level, level_axis=0) -> np.ndarray:
  """S = sum_k w_k * f64(y[k] + y[k+1]), the pair sum in y's dtype, summed in
  float64 from k = 0 upward and starting from the k = 0 term; 0 for fewer
  than 2 levels."""
  y = np.moveaxis(np.asarray(y), level_axis, 0)
  w = weights(level)
  if y.shape[0] < 2:
    return np.zeros(y.shape[1:])
  with np.errstate(invalid='ignore', over='ignore'):
    s = w[0] * (y[0] + y[1]).astype(np.float64)
    for k in range(1, y.shape[0] - 1):
      s = s + w[k] * (y[k] + y[k + 1]).astype(np.float64)
  return s


def window(level, level_min, level_max) -> slice:
  """`.sel(level=slice(level_min, level_max))` as pandas decides it."""
  return pd.Index(np.asarray(level)).slice_indexer(level_min, level_max)


def total_column(q, level, level_axis=0) -> np.ndarray:
  """(1 / 9.81) * S(q)."""
  return INV_G * level_sum(q, level, level_axis)


def ivt(q, u, v, level, level_axis=0, level_min=300, level_max=1000):
  """(1 / 9.81) * sqrt(S(q*u)^2 + S(q*v)^2) over the window; q*u in the
  common dtype of the three inputs."""
  dtype = np.result_type(q, u, v)
  q, u, v = (np.asarray(a, dtype) for a in (q, u, v))
  sl = window(level, level_min, level_max)
  take = lambda a: np.moveaxis(a, level_axis, 0)[sl]  # noqa: E731
  lev = np.asarray(level)[sl]
  with np.errstate(invalid='ignore', over='ignore'):
    su = level_sum(take(q) * take(u), lev)
    sv = level_sum(take(q) * take(v), lev)
    return INV_G * np.sqrt(su * su + sv * sv)


def zonal_anomaly(x, lon_axis):
  """f64(x) - the NaN-skipping zonal mean of x summed in float64 (NaN for an
  all-NaN row)."""
  x = np.asarray(x, np.float64)
  count = (~np.isnan(x)).sum(axis=lon_axis, keepdims=True)
  with np.errstate(invalid='ignore', divide='ignore'):
    mean = np.nansum(x, axis=lon_axis, keepdims=True) / count
  return x - mean


def eke(u, v, level, level_axis, lon_axis):
  """0.5 * S(u'^2 + v'^2), everything in float64."""
  du, dv = zonal_anomaly(u, lon_axis), zonal_anomaly(v, lon_axis)
  with np.errstate(invalid='ignore', over='ignore'):
    return 0.5 * level_sum(du * du + dv * dv, level, level_axis)


def eke_bound(u, v, level, level_axis, lon_axis):
  """The header's bound on |eke - reference| for float32 data:
  0.5 * sum_k |w_k| (e_k + e_{k+1}),
  e_k = 2^-23 (5 max y + 2 nlon (max|u'| max|u| + max|v'| max|v|)) over
  level k's row, NaN cells left out of the maxima."""
  nlon = np.shape(u)[lon_axis]
  du, dv = zonal_anomaly(u, lon_axis), zonal_anomaly(v, lon_axis)
  a = lambda x: np.abs(np.asarray(x, np.float64))  # noqa: E731
  with np.errstate(invalid='ignore'), warnings.catch_warnings():
    warnings.simplefilter('ignore', RuntimeWarning)  # all-NaN rows
    mx = lambda x: np.nan_to_num(np.nanmax(x, axis=lon_axis, keepdims=True))  # noqa: E731
    e = 2.0 ** -23 * (5 * mx(du * du + dv * dv) + 2 * nlon * (
        mx(a(du)) * mx(a(u)) + mx(a(dv)) * mx(a(v))))
  e = np.moveaxis(np.broadcast_to(e, np.shape(u)), level_axis, 0)
  w = np.abs(weights(level))
  out = np.zeros(e.shape[1:])
  for k in range(e.shape[0] - 1):
    out = out + w[k] * (e[k] + e[k + 1])
  return 0.5 * out


def sum_bound(y, level, level_axis=0) -> np.ndarray:
  """nlev * 2^-53 * sum_k |w_k p_k|: the reach of a reordered float64 level
  sum (NumPy's pairwise summation when `level` is the innermost axis)."""
  y = np.moveaxis(np.asarray(y), level_axis, 0)
  w = np.abs(weights(level))
  out = np.zeros(y.shape[1:])
  with np.errstate(invalid='ignore', over='ignore'):
    for k in range(y.shape[0] - 1):
      out = out + w[k] * np.abs((y[k] + y[k + 1]).astype(np.float64))
  return y.shape[0] * 2.0 ** -53 * out


def rounded(x, dtype) -> np.ndarray:
  """The one rounding of the float64 result to the data type."""
  return np.asarray(x, np.float64).astype(dtype)

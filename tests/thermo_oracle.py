"""The thermodynamic contract of include/wb2b200.h (wb2_lapse_rate,
wb2_relative_humidity) in NumPy: the lapse rate and relative humidity of
weatherbench2/derived_variables.py:341-362 and 433-468.  It does not import
the package.

Every function states the header's arithmetic step by step in the dtypes the
header names; tests/test_thermo_cpu.py pins it bit for bit to np.gradient and
to NumPy's own expressions."""
import numpy as np

INV_G = 1 / 9.81


def data_dtype(*arrays) -> np.dtype:
  """The common float type of the data: integers are taken as float64."""
  kinds = [np.float64 if np.asarray(a).dtype.kind in 'iu' else np.asarray(a).dtype
           for a in arrays]
  return np.result_type(*kinds)


def gradient(f, level, axis=0) -> np.ndarray:
  """np.gradient(f, level, edge_order=1, axis=axis) as the header states it:
  the differences in f's type, the level coordinate as float64, every
  derivative rounded once to f's type."""
  f = np.moveaxis(np.asarray(f), axis, 0)
  dtype = f.dtype
  x = np.asarray(level, np.float64)
  if x.size < 2 or f.shape[0] != x.size:
    raise ValueError('need at least 2 levels, one per index of the axis')
  dx = np.diff(x)
  tail = (None,) * (f.ndim - 1)
  out = np.empty(f.shape, dtype)
  with np.errstate(invalid='ignore', over='ignore', divide='ignore'):
    out[0] = ((f[1] - f[0]).astype(np.float64) / dx[0]).astype(dtype)
    out[-1] = ((f[-1] - f[-2]).astype(np.float64) / dx[-1]).astype(dtype)
    if (dx == dx[0]).all():
      mid = (f[2:] - f[:-2]).astype(np.float64) / (2. * dx[0])
    else:
      d1, d2 = dx[:-1][(slice(None),) + tail], dx[1:][(slice(None),) + tail]
      a = -d2 / (d1 * (d1 + d2))
      b = (d2 - d1) / (d1 * d2)
      c = d1 / (d2 * (d1 + d2))
      mid = (a * f[:-2].astype(np.float64) + b * f[1:-1].astype(np.float64)) + (
          c * f[2:].astype(np.float64))
    out[1:-1] = mid.astype(dtype)
  return np.moveaxis(out, 0, axis)


def lapse_rate(t, z, level, axis=0) -> np.ndarray:
  """dT / (T(1/9.81) * dZ) in the data type."""
  dtype = data_dtype(t, z)
  t, z = np.asarray(t, dtype), np.asarray(z, dtype)
  with np.errstate(invalid='ignore', over='ignore', divide='ignore'):
    dz = dtype.type(INV_G) * gradient(z, level, axis)
    return gradient(t, level, axis) / dz


def bolton_exp(x) -> np.ndarray:
  """exp of a float32 argument evaluated in float64 and rounded once; a
  float64 argument takes np.exp."""
  x = np.asarray(x)
  with np.errstate(over='ignore', invalid='ignore'):
    if x.dtype == np.float32:
      return np.exp(x.astype(np.float64)).astype(np.float32)
    return np.exp(x)


def bolton_argument(t) -> np.ndarray:
  """T(17.67) * (t - T(273.15)) / (t - T(29.65)) in t's type."""
  t = np.asarray(t)
  c = lambda v: t.dtype.type(v)  # noqa: E731
  with np.errstate(invalid='ignore', over='ignore', divide='ignore'):
    return c(17.67) * (t - c(273.15)) / (t - c(29.65))


def out_dtype(pressure, dtype) -> np.dtype:
  """NumPy's promotion of the pressure coordinate's dtype with the data's."""
  return np.result_type(np.asarray(pressure).dtype, dtype)


def relative_humidity(t, q, pressure, e=None, with_svp=False):
  """mr / (0.622 svp / (p - svp)) in the header's dtypes.  `pressure` is the
  coordinate in its own dtype, broadcastable against t; `e` replaces the
  rounded exp (to test the other float32 neighbour of a boundary case)."""
  dtype = data_dtype(t, q)
  t, q = np.asarray(t, dtype), np.asarray(q, dtype)
  o = out_dtype(pressure, dtype)
  c = lambda v: dtype.type(v)  # noqa: E731
  with np.errstate(invalid='ignore', over='ignore', divide='ignore'):
    e = bolton_exp(bolton_argument(t)) if e is None else np.asarray(e, dtype)
    svp = c(6.112) * e
    mr = q / (c(1) - q)
    smr = (c(0.622) * svp).astype(o) / (
        np.asarray(pressure).astype(o) - svp.astype(o))
    out = mr.astype(o) / smr
  return (out, svp) if with_svp else out


def exp_boundary(x):
  """For float32 arguments: the cells whose float64 exp lies within one
  float64 ulp of a float32 rounding boundary (where a faithfully rounded
  float64 exp may round the other way), and the other float32 value there."""
  x = np.asarray(x, np.float32)
  e64 = np.exp(x.astype(np.float64))
  e32 = e64.astype(np.float32)
  lo = np.nextafter(e64, -np.inf).astype(np.float32)
  hi = np.nextafter(e64, np.inf).astype(np.float32)
  flagged = (lo != e32) | (hi != e32)
  other = np.where(lo != e32, lo, hi)
  return flagged, other


def rh_bound(ref, svp, pressure, dtype) -> np.ndarray:
  """The header's bound on |out - NumPy's RH|:
  2^-20 |ref| (1 + |svp / (p - svp)|) for float32 data, 2^-49 (...) for
  float64."""
  eps = 2.0 ** -20 if np.dtype(dtype) == np.float32 else 2.0 ** -49
  svp = np.asarray(svp, np.float64)
  p = np.asarray(pressure, np.float64)
  with np.errstate(invalid='ignore', divide='ignore', over='ignore'):
    return eps * np.abs(np.asarray(ref, np.float64)) * (1 + np.abs(svp / (p - svp)))

"""TEST INFRASTRUCTURE: NumPy interpretation of wb2_column_integral
(include/wb2b200.h) on top of `fake_ctx.FakeContext`, so that the column
integrals run end to end on a CPU.  It reads the operands at the addresses,
strides, level count and weight table the operators hand to the library and
applies the header's arithmetic to them in float64 NumPy, so the CPU tests
check the pointer offsets, the tables and the layouts against
tests/column_oracle.py."""
import numpy as np

import fake_ctx
from fake_ctx import _view
from weatherbench2_b200 import _lib

INV_G = 1 / 9.81


def _level_sum(y, w):
  """sum_k w_k * f64(y[k] + y[k+1]) over axis 1, from k = 0 upward."""
  if y.shape[1] < 2:
    return np.zeros((y.shape[0],) + y.shape[2:])
  s = None
  for k in range(y.shape[1] - 1):
    term = w[k] * (y[:, k] + y[:, k + 1]).astype(np.float64)
    s = term if s is None else s + term
  return s


class ColumnFakeContext(fake_ctx.FakeContext):
  """FakeContext plus wb2_column_integral."""

  def column_integral(self, kind, dtype, q, u, v, nouter, outer_stride, nlev,
                      ninner, nlon, lon_stride, weight, out):
    self.calls.append(('column_integral', int(kind), int(dtype), int(nouter),
                       int(outer_stride), int(nlev), int(ninner), int(nlon),
                       int(lon_stride)))
    if kind not in (0, 1, 2) or dtype not in (_lib.F32, _lib.F64):
      raise _lib.Wb2Error('wb2_column_integral: unknown kind or dtype')
    if outer_stride < nlev * ninner:
      raise _lib.Wb2Error('wb2_column_integral: outer_stride too small')
    t = np.float64 if dtype == _lib.F64 else np.float32
    es = np.dtype(t).itemsize
    w = None if weight is None else np.asarray(weight, np.float64)
    assert nlev < 2 or w.shape == (nlev - 1,)

    def field(p):
      span = (nouter - 1) * outer_stride + nlev * ninner
      flat = _view(p, max(span, 0), t)
      return np.lib.stride_tricks.as_strided(
          flat, (nouter, nlev, ninner),
          (outer_stride * es, ninner * es, es)).copy()

    with np.errstate(invalid='ignore', over='ignore', divide='ignore'):
      if kind == 0:
        r = INV_G * _level_sum(field(q), w)
      elif kind == 1:
        qq = field(q)
        su = _level_sum(qq * field(u), w)
        sv = _level_sum(qq * field(v), w)
        r = INV_G * np.sqrt(su * su + sv * sv)
      else:
        assert ninner % nlon == 0
        nrow = ninner // nlon
        assert lon_stride in (1, nrow)
        shape = ((nouter, nlev, nrow, nlon) if lon_stride == 1
                 else (nouter, nlev, nlon, nrow))
        ax = 3 if lon_stride == 1 else 2

        def anomaly(x):
          x = x.reshape(shape).astype(np.float64)
          n = (~np.isnan(x)).sum(axis=ax, keepdims=True)
          return x - np.nansum(x, axis=ax, keepdims=True) / n

        du, dv = anomaly(field(u)), anomaly(field(v))
        y = (du * du + dv * dv).reshape(nouter, nlev, ninner)
        r = 0.5 * _level_sum(y, w)
    _view(out, nouter * ninner, t)[...] = np.asarray(r, t).reshape(-1)


def installed():
  """Makes `_lib.default_context()` return a ColumnFakeContext."""
  return fake_ctx.installed(ColumnFakeContext)

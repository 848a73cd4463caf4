"""TEST INFRASTRUCTURE: NumPy interpretation of wb2_lapse_rate and
wb2_relative_humidity (include/wb2b200.h) on top of `fake_ctx.FakeContext`, so
that the lapse rate and relative humidity run end to end on a CPU.  It reads
the operands at the addresses, sizes and host tables the operators hand to the
library -- the gradient coefficients for the lapse rate, the pressure table for
the relative humidity -- and applies the header's arithmetic to them, so the
CPU tests check the layouts, the tables and the dtypes against
tests/thermo_oracle.py."""
import numpy as np

import fake_ctx
import thermo_oracle as to
from fake_ctx import _view
from weatherbench2_b200 import _lib


def _type(code):
  if code not in (_lib.F32, _lib.F64):
    raise _lib.Wb2Error(f'unknown dtype {code}')
  return np.dtype(np.float64 if code == _lib.F64 else np.float32)


def _table_gradient(f, coef, uniform):
  """np.gradient along axis 1 of [nouter][nlev][ninner], from the header's
  coefficient table."""
  t = f.dtype
  c = np.asarray(coef, np.float64)
  out = np.empty_like(f)
  n = f.shape[1]
  with np.errstate(invalid='ignore', over='ignore', divide='ignore'):
    out[:, 0] = ((f[:, 1] - f[:, 0]).astype(np.float64) / c[0, 0]).astype(t)
    out[:, -1] = ((f[:, -1] - f[:, -2]).astype(np.float64) / c[-1, 0]).astype(t)
    for k in range(1, n - 1):
      if uniform:
        r = (f[:, k + 1] - f[:, k - 1]).astype(np.float64) / c[k, 0]
      else:
        r = (c[k, 0] * f[:, k - 1].astype(np.float64) +
             c[k, 1] * f[:, k].astype(np.float64)) + (
                 c[k, 2] * f[:, k + 1].astype(np.float64))
      out[:, k] = r.astype(t)
  return out


class ThermoFakeContext(fake_ctx.FakeContext):
  """FakeContext plus wb2_lapse_rate and wb2_relative_humidity."""

  def lapse_rate(self, dtype, t, z, nouter, nlev, ninner, coef, uniform, out):
    self.calls.append(('lapse_rate', int(dtype), int(nouter), int(nlev),
                       int(ninner), bool(uniform)))
    ty = _type(dtype)
    if nlev < 2:
      raise _lib.Wb2Error('wb2_lapse_rate: need at least 2 levels')
    assert np.shape(coef) == (nlev, 3)
    n = nouter * nlev * ninner
    shape = (nouter, nlev, ninner)
    tt = _view(t, n, ty).reshape(shape)
    zz = _view(z, n, ty).reshape(shape)
    with np.errstate(invalid='ignore', over='ignore', divide='ignore'):
      dz = ty.type(to.INV_G) * _table_gradient(zz, coef, uniform)
      r = _table_gradient(tt, coef, uniform) / dz
    _view(out, n, ty)[...] = r.reshape(-1)

  def relative_humidity(self, dtype, out_dtype, t, q, nouter, npres, ninner,
                        pressure, out):
    self.calls.append(('relative_humidity', int(dtype), int(out_dtype),
                       int(nouter), int(npres), int(ninner)))
    ty, oy = _type(dtype), _type(out_dtype)
    if ty == np.float64 and oy == np.float32:
      raise _lib.Wb2Error('wb2_relative_humidity: out_dtype narrower than data')
    p = np.asarray(pressure, np.float64)
    assert p.shape == (npres,)
    n = nouter * npres * ninner
    shape = (nouter, npres, ninner)
    r = to.relative_humidity(_view(t, n, ty).reshape(shape),
                             _view(q, n, ty).reshape(shape),
                             p.astype(oy)[None, :, None])
    assert r.dtype == oy
    _view(out, n, oy)[...] = r.reshape(-1)


def installed():
  """Makes `_lib.default_context()` return a ThermoFakeContext."""
  return fake_ctx.installed(ThermoFakeContext)

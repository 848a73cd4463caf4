"""TEST INFRASTRUCTURE: NumPy interpretation of wb2_wind_dynamics
(include/wb2b200.h) on top of `fake_ctx.FakeContext`, so that the wind
dynamics derived variables run end to end on a CPU.  It reads the fields, the
strides and the gradient-coefficient / cos / Coriolis / pressure tables the
operators hand to the library and applies the header's arithmetic to them in
float64 NumPy (which never fuses a multiply-add), so the CPU tests check both
the tables and the arithmetic contract against tests/dynamics_oracle.py."""
import numpy as np

import fake_ctx
from fake_ctx import _view
from weatherbench2_b200 import _lib

M = 2 * np.pi * (1000 * (6357 + 6378) / 2) / 360


def table_gradient(f, table, uniform):
  """np.gradient along the last axis of float32 `f` from an [n][3] table."""
  f = np.asarray(f, np.float32)
  t = np.asarray(table, np.float64)
  out = np.empty(f.shape, np.float32)
  with np.errstate(invalid='ignore', over='ignore'):
    out[..., 0] = (f[..., 1] - f[..., 0]).astype(np.float64) / t[0, 0]
    out[..., -1] = (f[..., -1] - f[..., -2]).astype(np.float64) / t[-1, 0]
    if uniform:
      out[..., 1:-1] = (f[..., 2:] - f[..., :-2]).astype(np.float64) / t[1:-1, 0]
    else:
      out[..., 1:-1] = (t[1:-1, 0] * f[..., :-2].astype(np.float64) +
                        t[1:-1, 1] * f[..., 1:-1].astype(np.float64) +
                        t[1:-1, 2] * f[..., 2:].astype(np.float64))
  return out


def interpret(kind, u, v, z, lat_coef, lat_uniform, lon_coef, lon_uniform,
              cos_lat, coriolis, pressure):
  """The header's arithmetic on [nouter][nlev][nlat][nlon] float32 fields;
  float32 result."""
  cos = np.asarray(cos_lat, np.float64)[:, None]

  def ddx(f):
    g = table_gradient(f, lon_coef, lon_uniform).astype(np.float64)
    with np.errstate(divide='ignore', invalid='ignore'):
      return np.where(cos > 1e-6, g / cos / M, 0.0)

  def ddy(f):
    g = table_gradient(np.swapaxes(f, -1, -2), lat_coef, lat_uniform)
    return np.swapaxes(g, -1, -2) / np.float32(M)

  with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
    if kind in (0, 2):
      r = ddx(u) + ddy(v).astype(np.float64)
      if kind == 2:
        p = np.asarray(pressure, np.float64)
        acc = np.zeros(r.shape)
        run = None
        for k in range(1, r.shape[1]):
          term = (p[k] - p[k - 1]) * (-r[:, k] + -r[:, k - 1]) / 2.0
          run = term if run is None else run + term
          acc[:, k] = run
        r = acc
    elif kind == 1:
      r = ddx(v) - ddy(u).astype(np.float64)
    else:
      f = np.asarray(coriolis, np.float64)[:, None]
      ug = (-ddy(z)).astype(np.float64) / f
      vg = ddx(z) / f
      if kind in (6, 7, 8):
        ua = (u.astype(np.float64) - ug) if u is not None else None
        va = (v.astype(np.float64) - vg) if v is not None else None
      r = {3: lambda: np.sqrt(ug * ug + vg * vg), 4: lambda: ug,
           5: lambda: vg, 6: lambda: np.sqrt(ua * ua + va * va),
           7: lambda: ua, 8: lambda: va}[kind]()
  return r.astype(np.float32)


class DynamicsFakeContext(fake_ctx.FakeContext):
  """FakeContext plus wb2_wind_dynamics."""

  def wind_dynamics(self, kind, u, v, z, nouter, nlev, nlat, nlon, lat_stride,
                    lon_stride, lat_coef, lat_uniform, lon_coef, lon_uniform,
                    cos_lat, coriolis, pressure, out):
    self.calls.append(('wind_dynamics', int(kind), int(nouter), int(nlev),
                       int(nlat), int(nlon), int(lat_stride), int(lon_stride)))
    if nlat < 2 or nlon < 2:
      raise _lib.Wb2Error('wb2_wind_dynamics: need at least 2 points')
    assert (lat_stride, lon_stride) in ((nlon, 1), (1, nlat))
    lon_contig = lon_stride == 1
    n = nouter * nlev * nlat * nlon

    def field(p):
      if not p:
        return None
      x = _view(p, n, np.float32)
      if lon_contig:
        return x.reshape(nouter, nlev, nlat, nlon)
      return np.swapaxes(x.reshape(nouter, nlev, nlon, nlat), -1, -2)

    r = interpret(int(kind), field(u), field(v), field(z),
                  np.asarray(lat_coef).reshape(nlat, 3), lat_uniform,
                  np.asarray(lon_coef).reshape(nlon, 3), lon_uniform, cos_lat,
                  coriolis, pressure)
    if not lon_contig:
      r = np.swapaxes(r, -1, -2)
    _view(out, n, np.float32)[...] = r.reshape(-1)


def installed():
  """Makes `_lib.default_context()` return a DynamicsFakeContext."""
  return fake_ctx.installed(DynamicsFakeContext)

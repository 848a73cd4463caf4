#!/usr/bin/env python
"""Runs the REFERENCE's own wind-dynamics derived variables
(<reference>/weatherbench2/derived_variables.py:102-338: divergence, vorticity,
vertical velocity, geostrophic and ageostrophic winds -- imported, not copied)
on the seeded cases below and stores their inputs and results in
reference_dynamics_vectors.npz.

Like make_reference_vectors.py, the reference module executes on
tests/golden/xarray_shim.  `extend_shim` adds the xarray calls these classes
make and the other reference modules do not: `DataArray.differentiate`
(np.gradient with the coordinate as sample points), unary `+`, and ufuncs /
arithmetic on a coordinate, which is a DataArray in xarray.  tests/test_wind_dynamics_cpu.py holds
tests/dynamics_oracle.py and the operators (on a NumPy interpretation of the
C ABI) to the committed vectors; only this script reads the reference.

Run:  python tests/golden/make_dynamics_vectors.py <reference checkout>
"""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(HERE, 'xarray_shim'),
                os.path.abspath(sys.argv[1]) if len(sys.argv) > 1 else '']

KINDS = ('divergence', 'vorticity', 'vertical_velocity',
         'geostrophic_wind_speed', 'u_component_of_geostrophic_wind',
         'v_component_of_geostrophic_wind', 'ageostrophic_wind_speed',
         'u_component_of_ageostrophic_wind', 'v_component_of_ageostrophic_wind')


def extend_shim(xr):
  """The xarray calls of derived_variables.py:102-338 the shim lacks, each
  written to xarray's documented semantics."""
  import weatherbench2_b200.xarray_lite as xl
  da_cls = xr.DataArray

  def differentiate(self, coord, edge_order=1, datetime_unit=None):
    # xarray/core/dataarray.py -> duck_array_ops.gradient: np.gradient on the
    # coordinate's values; the result keeps the data's dtype
    del datetime_unit
    ax = self.dims.index(coord)
    grad = np.gradient(np.asarray(self.values),
                       np.asarray(self.coords[coord].values),
                       edge_order=edge_order, axis=ax)
    return self._replace(grad)  # pylint: disable=protected-access

  def coord_da(c):
    return da_cls(c.values, c.dims,
                  {c.dims[0]: c.values} if len(c.dims) == 1 else None)

  def coord_ufunc(self, ufunc, method, *inputs, **kwargs):
    del self
    args = [coord_da(i) if isinstance(i, xl.Coord) else i for i in inputs]
    return getattr(ufunc, method)(*args, **kwargs)

  da_cls.differentiate = differentiate
  da_cls.__pos__ = lambda self: self._replace(+np.asarray(self.values))  # pylint: disable=protected-access
  xl.Coord.__array_ufunc__ = coord_ufunc
  for op in ('__add__', '__radd__', '__sub__', '__rsub__', '__mul__',
             '__rmul__', '__truediv__', '__rtruediv__', '__neg__', '__gt__'):
    setattr(xl.Coord, op,
            lambda self, *o, _op=op: getattr(coord_da(self), _op)(*o))


def cases():
  """name -> (dims, latitude, longitude, level, seed)."""
  lat_nu = np.sort(np.r_[np.linspace(-90, 90, 11), 0.0, 7.5])
  lon_nu = np.cumsum(np.r_[0.0, np.tile([20.0, 25.0], 7)])
  tlll = ('time', 'level', 'latitude', 'longitude')
  return {
      'uniform': (tlll, np.linspace(-90, 90, 13), np.arange(16) * 22.5,
                  (1000, 850, 500), 0),
      'nonuniform': (tlll, lat_nu, lon_nu, (1000, 700, 250), 1),
      'descending_lat': (tlll, np.linspace(90, -90, 11), np.arange(12) * 30.0,
                         (50, 500, 1000), 2),
      'regional': (tlll, np.linspace(25, 65, 9), np.linspace(-30, 30, 13),
                   (850, 500, 200), 3),
      'lon_lat_layout': (('level', 'time', 'longitude', 'latitude'),
                         np.linspace(-90, 90, 13), np.arange(16) * 22.5,
                         (1000, 850, 500), 4),
  }


def inputs(dims, lat, lon, level, seed):
  sizes = {'time': 1, 'level': len(level), 'latitude': lat.size,
           'longitude': lon.size}
  shape = tuple(sizes[d] for d in dims)
  rs = np.random.RandomState(seed)
  u = rs.normal(scale=10, size=shape).astype(np.float32)
  v = rs.normal(scale=10, size=shape).astype(np.float32)
  z = (5e4 + rs.normal(scale=300, size=shape)).astype(np.float32)
  u.reshape(-1)[5] = np.nan
  z.reshape(-1)[shape[-1] + 2] = np.nan
  return u, v, z


def main():
  import xarray as xr  # the shim
  extend_shim(xr)
  from weatherbench2 import derived_variables
  out = {}
  for name, (dims, lat, lon, level, seed) in cases().items():
    u, v, z = inputs(dims, lat, lon, level, seed)
    ds = xr.Dataset(
        {'u_component_of_wind': (dims, u), 'v_component_of_wind': (dims, v),
         'geopotential': (dims, z)},
        {'time': np.arange(1), 'level': np.asarray(level), 'latitude': lat,
         'longitude': lon})
    out[f'{name}|u'], out[f'{name}|v'], out[f'{name}|z'] = u, v, z
    out[f'{name}|dims'] = np.array(dims)
    out[f'{name}|latitude'], out[f'{name}|longitude'] = lat, lon
    out[f'{name}|level'] = np.asarray(level)
    for kind in KINDS:
      with warnings.catch_warnings():
        warnings.simplefilter('ignore', RuntimeWarning)
        res = derived_variables.DERIVED_VARIABLE_DICT[kind].compute(ds)
      out[f'{name}|{kind}'] = np.asarray(res.transpose(*dims).values)
      print('ran', name, kind, res.dtype)
  np.savez_compressed(os.path.join(HERE, 'reference_dynamics_vectors.npz'),
                      **out)


if __name__ == '__main__':
  main()

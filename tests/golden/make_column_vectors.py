#!/usr/bin/env python
"""Runs the REFERENCE's own column-integral derived variables
(<reference>/weatherbench2/derived_variables.py:212-228 and 365-430:
EddyKineticEnergy, TotalColumnWater, IntegratedWaterTransport -- imported, not
copied) on the seeded cases below and stores their inputs and results in
reference_column_vectors.npz.

Like make_dynamics_vectors.py, the reference module executes on
tests/golden/xarray_shim.  `extend_shim` replaces the shim's
`DataArray.integrate` with xarray's own arithmetic (duck_array_ops.trapz:
sum(dx * 0.5 * (y[1:] + y[:-1]), skipna=False) with dx in the coordinate's
dtype) at run time; the zonal `mean` is the shim's, which skips NaN as
xarray's does.  The shim's files are unchanged.  tests/test_column_integrals_cpu.py
holds tests/column_oracle.py and the operators (on a NumPy interpretation of
the C ABI) to the committed vectors; only this script reads the reference.

Run:  python tests/golden/make_column_vectors.py <reference checkout>
"""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(HERE, 'xarray_shim'),
                os.path.abspath(sys.argv[1]) if len(sys.argv) > 1 else '']

# name in the npz -> (DERIVED_VARIABLE_DICT entry or None, class kwargs)
KINDS = {
    'total_column_vapor': ('total_column_vapor', None),
    'total_column_liquid': ('total_column_liquid', None),
    'total_column_ice': ('total_column_ice', None),
    'integrated_vapor_transport': ('integrated_vapor_transport', None),
    'ivt_all_levels': (None, dict(level_min=None, level_max=None)),
    'ivt_narrow': (None, dict(level_min=500, level_max=850)),
    'ivt_empty': (None, dict(level_min=1000, level_max=300)),
    'eddy_kinetic_energy': ('eddy_kinetic_energy', None),
}
SPECIES = ('specific_humidity', 'specific_cloud_liquid_water_content',
           'specific_cloud_ice_water_content')


def extend_shim(xr):
  """xarray's integrate (Dataset._integrate_one -> duck_array_ops.trapz)."""

  def integrate(self, coord):
    ax = self.dims.index(coord)
    y = np.asarray(self.values)
    x = np.asarray(self.coords[coord].values)
    tail = (None,) * (y.ndim - ax - 1)
    dx = x[(slice(1, None),) + tail] - x[(slice(None, -1),) + tail]
    lo = (slice(None),) * ax + (slice(1, None),)
    hi = (slice(None),) * ax + (slice(None, -1),)
    integrand = dx * 0.5 * (y[lo] + y[hi])
    keep = tuple(d for d in self.dims if d != coord)
    return self._replace(np.sum(integrand, axis=ax), keep)  # pylint: disable=protected-access

  xr.DataArray.integrate = integrate


def cases():
  """name -> (dims, level, latitude, longitude, seed)."""
  tlll = ('time', 'level', 'latitude', 'longitude')
  return {
      'ascending': (tlll, (50, 100, 250, 300, 500, 700, 850, 925, 1000),
                    np.linspace(-90, 90, 7), np.arange(12) * 30.0, 0),
      'descending': (tlll, (1000, 850, 700, 500, 300, 50),
                     np.linspace(-90, 90, 5), np.arange(8) * 45.0, 1),
      'nonuniform': (tlll, (100, 137.5, 300, 312.25, 500, 1000),
                     np.linspace(-90, 90, 5), np.arange(10) * 36.0, 2),
      'single_level': (tlll, (500,), np.linspace(-90, 90, 5),
                       np.arange(8) * 45.0, 3),
      'level_innermost': (('time', 'latitude', 'longitude', 'level'),
                          (100, 300, 500, 700, 850, 1000),
                          np.linspace(-90, 90, 5), np.arange(8) * 45.0, 4),
      'lon_lat_layout': (('time', 'level', 'longitude', 'latitude'),
                         (200, 300, 500, 850, 1000), np.linspace(-90, 90, 6),
                         np.arange(9) * 40.0, 5),
      'regional': (tlll, (300, 400, 500, 600, 700, 850, 1000),
                   np.linspace(25, 65, 9), np.linspace(-30, 30, 13), 6),
  }


def inputs(dims, level, lat, lon, seed):
  sizes = {'time': 2, 'level': len(level), 'latitude': lat.size,
           'longitude': lon.size}
  shape = tuple(sizes[d] for d in dims)
  rs = np.random.RandomState(seed)
  out = {}
  for i, name in enumerate(SPECIES):
    out[name] = (np.abs(rs.normal(scale=4e-3 / (i + 1), size=shape))
                 .astype(np.float32))
  out['u_component_of_wind'] = (5 + rs.normal(scale=12, size=shape)).astype(
      np.float32)
  out['v_component_of_wind'] = rs.normal(scale=8, size=shape).astype(
      np.float32)
  # a NaN cell in q and u, and one zonal row of v that is NaN throughout
  out['specific_humidity'].reshape(-1)[3] = np.nan
  out['u_component_of_wind'].reshape(-1)[7] = np.nan
  lon_ax, lat_ax = dims.index('longitude'), dims.index('latitude')
  row = [0] * len(dims)
  row[lon_ax] = slice(None)
  row[lat_ax] = 1
  out['v_component_of_wind'][tuple(row)] = np.nan
  return out


def main():
  import xarray as xr  # the shim
  extend_shim(xr)
  from weatherbench2 import derived_variables
  out = {}
  for name, (dims, level, lat, lon, seed) in cases().items():
    fields = inputs(dims, level, lat, lon, seed)
    ds = xr.Dataset({k: (dims, a) for k, a in fields.items()},
                    {'time': np.arange(2), 'level': np.asarray(level),
                     'latitude': lat, 'longitude': lon})
    for k, a in fields.items():
      out[f'{name}|{k}'] = a
    out[f'{name}|dims'] = np.array(dims)
    out[f'{name}|level'] = np.asarray(level)
    out[f'{name}|latitude'], out[f'{name}|longitude'] = lat, lon
    for kind, (entry, kwargs) in KINDS.items():
      var = (derived_variables.DERIVED_VARIABLE_DICT[entry] if entry else
             derived_variables.IntegratedWaterTransport(**kwargs))
      with warnings.catch_warnings():
        warnings.simplefilter('ignore', RuntimeWarning)
        res = var.compute(ds)
      keep = tuple(d for d in dims if d != 'level')
      out[f'{name}|{kind}'] = np.asarray(res.transpose(*keep).values)
      print('ran', name, kind, res.dtype, res.dims)
  np.savez_compressed(os.path.join(HERE, 'reference_column_vectors.npz'),
                      **out)


if __name__ == '__main__':
  main()

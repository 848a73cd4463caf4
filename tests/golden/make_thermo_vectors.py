#!/usr/bin/env python
"""Runs the REFERENCE's own thermodynamic derived variables
(<reference>/weatherbench2/derived_variables.py:341-362 and 433-468: LapseRate,
RelativeHumidity -- imported, not copied) on the seeded cases below and stores
their inputs and results in reference_thermo_vectors.npz.

Like make_dynamics_vectors.py, the reference module executes on
tests/golden/xarray_shim, extended at run time by that script's
`extend_shim`: `DataArray.differentiate` (np.gradient with the coordinate as
sample points) and arithmetic on a coordinate, which is a DataArray in xarray.
The shim's files are unchanged.  tests/test_thermo_cpu.py holds
tests/thermo_oracle.py and the operators (on a NumPy interpretation of the C
ABI) to the committed vectors; only this script reads the reference.

The `metpy` case is the input of the reference's
derived_variables_test.py::testRelativeHumidity; its MetPy answer is stored as
`metpy|expected` (compared with atol 1e-4).

Run:  python tests/golden/make_thermo_vectors.py <reference checkout>
"""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, HERE, os.path.join(HERE, 'xarray_shim'),
                os.path.abspath(sys.argv[1]) if len(sys.argv) > 1 else '']

WB2_LEVELS = (50, 100, 150, 200, 250, 300, 400, 500, 600, 700, 850, 925, 1000)
METPY_EXPECTED = np.array([0.2116, 0.3115, 0.5937, 0.8462])


def cases():
  """name -> (dims, level, seed)."""
  tlll = ('time', 'level', 'latitude', 'longitude')
  return {
      'wb2_ascending': (tlll, np.array(WB2_LEVELS), 0),
      'wb2_descending': (('level', 'time', 'longitude', 'latitude'),
                         np.array(WB2_LEVELS[::-1]), 1),
      'uniform_3': (('time', 'latitude', 'longitude', 'level'),
                    np.array([500, 700, 900]), 2),
      'two_levels': (tlll, np.array([850, 1000]), 3),
      'float32_levels': (tlll, np.array([200, 300, 500, 700, 850, 925, 1000],
                                        np.float32), 4),
  }


def standard_height(level):
  """Height in m of a pressure level in the standard atmosphere."""
  return 44330.8 * (1 - (np.asarray(level, np.float64) / 1013.25) ** 0.190263)


def inputs(dims, level, seed):
  """Temperature, geopotential and specific humidity with realistic vertical
  profiles, NaN cells, and one column whose geopotential is constant
  (dz == 0, so the lapse rate is +-inf or NaN there)."""
  sizes = {'time': 2, 'level': len(level), 'latitude': 5, 'longitude': 8}
  shape = tuple(sizes[d] for d in dims)
  rs = np.random.RandomState(seed)
  prof = [None] * len(dims)
  prof[dims.index('level')] = slice(None)
  h = standard_height(level)[tuple(prof)]
  temp = (288.15 - 6.5e-3 * np.minimum(h, 11000) +
          rs.normal(scale=3, size=shape)).astype(np.float32)
  geo = (9.81 * h + rs.normal(scale=40, size=shape)).astype(np.float32)
  q = (np.abs(rs.normal(scale=6e-3, size=shape)) *
       np.exp(-h / 2500)).astype(np.float32)
  temp.reshape(-1)[3] = np.nan
  geo.reshape(-1)[11] = np.nan
  q.reshape(-1)[5] = np.nan
  col = [0] * len(dims)
  col[dims.index('level')] = slice(None)
  col[dims.index('longitude')] = 2
  geo[tuple(col)] = geo[tuple(col)][0]
  return {'temperature': temp, 'geopotential': geo, 'specific_humidity': q}


def main():
  import xarray as xr  # the shim
  from make_dynamics_vectors import extend_shim
  extend_shim(xr)
  from weatherbench2 import derived_variables
  out = {}
  for name, (dims, level, seed) in cases().items():
    fields = inputs(dims, level, seed)
    ds = xr.Dataset({k: (dims, a) for k, a in fields.items()},
                    {'time': np.arange(2), 'level': level,
                     'latitude': np.linspace(-60, 60, 5),
                     'longitude': np.arange(8) * 45.0})
    for k, a in fields.items():
      out[f'{name}|{k}'] = a
    out[f'{name}|dims'] = np.array(dims)
    out[f'{name}|level'] = level
    for kind, var in (('lapse_rate', derived_variables.LapseRate()),
                      ('relative_humidity',
                       derived_variables.RelativeHumidity())):
      with warnings.catch_warnings():
        warnings.simplefilter('ignore', RuntimeWarning)
        res = var.compute(ds)
      out[f'{name}|{kind}'] = np.asarray(res.transpose(*dims).values)
      print('ran', name, kind, res.dtype, res.dims)
  # derived_variables_test.py::testRelativeHumidity
  ds = xr.Dataset(
      {'temperature': ('level', np.array([240, 280, 295, 310])),
       'specific_humidity': ('level', np.array([1e-3, 1e-2, 2e-2, 4e-2]))},
      coords={'level': np.array([50, 200, 500, 850])})
  res = derived_variables.RelativeHumidity().compute(ds)
  for k in ('temperature', 'specific_humidity', 'level'):
    out[f'metpy|{k}'] = np.asarray(ds[k].values)
  out['metpy|dims'] = np.array(('level',))
  out['metpy|relative_humidity'] = np.asarray(res.values)
  out['metpy|expected'] = METPY_EXPECTED
  print('ran metpy relative_humidity', res.dtype, res.dims)
  np.savez_compressed(os.path.join(HERE, 'reference_thermo_vectors.npz'),
                      **out)


if __name__ == '__main__':
  main()

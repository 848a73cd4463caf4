#!/usr/bin/env python
"""Runs the REFERENCE's own `moment_reduce`
(<reference>/scripts/compute_statistical_moments.py:47-79 -- imported, not
copied) for the zeroth, first and second orders, and the weighting step of
<reference>/scripts/compute_averages.py:137-152 (`metrics.get_lat_weights`
times the data), on the seeded fields below.  It stores their inputs and
results in reference_moment_vectors.npz.

Like make_precip_vectors.py, the reference modules execute on
tests/golden/xarray_shim, where absl is real and apache_beam / xarray_beam are
import stubs.  `extend_shim` adds the one call they make that the shim lacks,
`DataArray.reindex_like` (an identity here: the weights already share the
data's latitude coordinate).  `xbeam.Mean` cannot run on the stub, so the
average vectors store the reference's weighted product reduced by sum / count
in float64, which is what that Mean computes.  tests/test_average_golden.py
holds the operators (on a NumPy interpretation of the C ABI) to the committed
vectors; only this script reads the reference.

Run:  python tests/golden/make_moment_vectors.py <reference checkout>
"""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(HERE, 'xarray_shim'),
                os.path.abspath(sys.argv[1]) if len(sys.argv) > 1 else '']

DIMS = ('time', 'level', 'longitude', 'latitude')


def extend_shim(xr):
  xr.DataArray.reindex_like = lambda self, other, **kw: self


def field(seed, dtype):
  """[time 5][level 2][longitude 9][latitude 7] with 10 % NaN, an all-NaN
  time step and a fully valid level."""
  rs = np.random.RandomState(seed)
  x = (280.0 + 20.0 * rs.standard_normal((5, 2, 9, 7))).astype(dtype)
  x[rs.uniform(size=x.shape) < 0.1] = np.nan
  x[2] = np.nan
  x[4, 1] = 280.0 + rs.standard_normal((9, 7))
  return x


def coords():
  return {'time': np.arange(5), 'level': np.array([500.0, 850.0]),
          'longitude': np.arange(9) * 40.0,
          'latitude': np.linspace(-90.0, 90.0, 7)}


def main():
  import xarray as xr  # the shim
  extend_shim(xr)
  from scripts import compute_statistical_moments as csm
  from weatherbench2 import metrics
  out = {}
  for seed, dtype in ((0, np.float32), (1, np.float64)):
    tag = np.dtype(dtype).name
    x = field(seed, dtype)
    ds = xr.Dataset({'t': (DIMS, x)}, coords())
    out[f'{tag}|x'] = x
    for reduce_dims in (('longitude', 'latitude'), ('time',)):
      key = f'{tag}|{"_".join(reduce_dims)}'
      for order in ('zeroth', 'first', 'second'):
        with warnings.catch_warnings():
          warnings.simplefilter('ignore', RuntimeWarning)
          res = csm.moment_reduce(ds, order=order, reduce_dims=reduce_dims)
        keep = tuple(d for d in DIMS if d not in reduce_dims)
        out[f'{key}|{order}'] = np.asarray(res['t'].transpose(*keep).values)
        print('ran', key, order, res['t'].dtype, res['t'].dims)
    # compute_averages.py: v * weights.reindex_like(v), then the Mean
    weights = metrics.get_lat_weights(ds)
    wx = np.asarray((ds['t'] * weights.reindex_like(ds['t']))
                    .transpose(*DIMS).values)
    out[f'{tag}|lat_weights'] = np.asarray(weights.values)
    for avg, axes in ((('time', 'latitude'), (0, 3)),
                      (('longitude', 'latitude'), (2, 3))):
      key = f'{tag}|avg|{"_".join(avg)}'
      with warnings.catch_warnings():
        warnings.simplefilter('ignore', RuntimeWarning)
        out[f'{key}|skipna'] = (np.nansum(wx, axis=axes) /
                                (~np.isnan(wx)).sum(axis=axes))
        out[f'{key}|noskip'] = wx.sum(axis=axes) / np.prod(
            [wx.shape[a] for a in axes])
  np.savez_compressed(os.path.join(HERE, 'reference_moment_vectors.npz'),
                      **out)


if __name__ == '__main__':
  main()

#!/usr/bin/env python
"""Runs the REFERENCE's own precipitation accumulations
(<reference>/weatherbench2/derived_variables.py:471-528, 685-720:
PrecipitationAccumulation and AggregatePrecipitationAccumulation -- imported,
not copied) on the seeded cases below and stores their inputs and results in
reference_precip_vectors.npz.

Like make_dynamics_vectors.py, the reference module executes on
tests/golden/xarray_shim.  `extend_shim` adds the xarray calls these classes
make and the shim lacks, each written to xarray's documented semantics:
`DataArray.diff` (n=1, label='upper', in the data's dtype),
`DataArray.rolling({dim: w}).sum()` (min_periods = w; the window summed in
the data's dtype, oldest first, as bottleneck's move_sum does for a fresh
window), `DataArray.where(cond, other)` and comparisons with scalars.
tests/test_precip_accumulation_cpu.py holds tests/precip_oracle.py and the
operators to the committed vectors within the documented float32 bound; only
this script reads the reference.

Run:  python tests/golden/make_precip_vectors.py <reference checkout>
"""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(HERE, 'xarray_shim'),
                os.path.abspath(sys.argv[1]) if len(sys.argv) > 1 else '']

LEAD = 'prediction_timedelta'


def extend_shim(xr):
  da_cls = xr.DataArray

  def diff(self, dim, n=1, label='upper'):
    assert n == 1 and label == 'upper'
    ax = self.dims.index(dim)
    vals = np.diff(np.asarray(self.values), axis=ax)
    coords = {k: c for k, c in self.coords.items() if dim not in c.dims}
    coords[dim] = np.asarray(self.coords[dim].values)[1:]
    return da_cls(vals, self.dims, coords, self.name, self.attrs)

  class _Rolling:

    def __init__(self, da, windows):
      (self.dim, self.w), = windows.items()
      self.da = da

    def sum(self):
      da, w = self.da, self.w
      ax = da.dims.index(self.dim)
      x = np.moveaxis(np.asarray(da.values), ax, -1)
      out = np.full(x.shape, np.nan, x.dtype)
      for t in range(w - 1, x.shape[-1]):
        s = x[..., t - w + 1]
        for k in range(t - w + 2, t + 1):
          s = s + x[..., k]
        out[..., t] = s
      return da_cls(np.moveaxis(out, -1, ax), da.dims, dict(da.coords),
                    da.name, da.attrs)

  def where(self, cond, other):
    c = np.asarray(cond.values if hasattr(cond, 'values') else cond)
    vals = np.where(c, np.asarray(self.values), other)
    return da_cls(vals, self.dims, dict(self.coords), self.name, self.attrs)

  da_cls.diff = diff
  da_cls.rolling = lambda self, windows: _Rolling(self, windows)
  da_cls.where = where


def cases():
  """name -> (class, kwargs, dims, lead (hours), seed, kind)."""
  return {
      'tp6_w1': ('PrecipitationAccumulation', dict(accumulation_hours=6),
                 ('time', LEAD, 'latitude'), np.arange(0, 66, 6), 0, 'tp'),
      'tp24_w4': ('PrecipitationAccumulation', dict(accumulation_hours=24),
                  ('time', LEAD, 'latitude'), np.arange(0, 66, 6), 1, 'tp'),
      'tp24_hourly_lead_last': ('PrecipitationAccumulation',
                                dict(accumulation_hours=24),
                                ('latitude', 'time', LEAD), np.arange(0, 49),
                                2, 'tp'),
      'tp12_noclamp': ('PrecipitationAccumulation',
                       dict(accumulation_hours=12, set_negative_to_zero=False),
                       (LEAD, 'latitude'), np.arange(0, 72, 6), 3, 'tp'),
      'agg24_from_6': ('AggregatePrecipitationAccumulation',
                       dict(accumulation_hours=24),
                       ('time', LEAD, 'latitude'), np.arange(0, 66, 6), 4,
                       'acc'),
  }


def inputs(dims, nlead, seed, kind):
  sizes = {'time': 2, LEAD: nlead, 'latitude': 5}
  shape = tuple(sizes[d] for d in dims)
  rs = np.random.RandomState(seed)
  ax = dims.index(LEAD)
  steps = rs.exponential(2e-3, size=shape).astype(np.float32)
  # a few small negative steps, as models produce
  steps[rs.uniform(size=shape) < 0.15] *= -0.05
  if kind == 'acc':
    return steps
  tp = np.cumsum(steps, axis=ax, dtype=np.float32)
  tp.reshape(-1)[7] = np.nan
  return tp


def main():
  import xarray as xr  # the shim
  extend_shim(xr)
  from weatherbench2 import derived_variables
  out = {}
  for name, (cls, kwargs, dims, hours, seed, kind) in cases().items():
    lead = hours.astype('timedelta64[h]').astype('timedelta64[ns]')
    x = inputs(dims, lead.size, seed, kind)
    var = ('total_precipitation' if kind == 'tp' else
           'total_precipitation_6hr')
    coords = {LEAD: lead, 'time': np.arange(2), 'latitude': np.arange(5.0)}
    ds = xr.Dataset({var: (dims, x)},
                    {k: v for k, v in coords.items() if k in dims})
    if kind == 'tp':
      obj = getattr(derived_variables, cls)(total_precipitation_name=var,
                                            **kwargs)
    else:
      obj = getattr(derived_variables, cls)(**kwargs)
    with warnings.catch_warnings():
      warnings.simplefilter('ignore', RuntimeWarning)
      res = obj.compute(ds)
    out[f'{name}|x'] = x
    out[f'{name}|dims'] = np.array(dims)
    out[f'{name}|lead_hours'] = hours
    out[f'{name}|result'] = np.asarray(res.transpose(*dims).values)
    print('ran', name, res.dtype, res.dims)
  np.savez_compressed(os.path.join(HERE, 'reference_precip_vectors.npz'),
                      **out)


if __name__ == '__main__':
  main()

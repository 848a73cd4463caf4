"""CPU tests of moment_reduce and compute_averages against vectors from the
reference's own code (tests/golden/reference_moment_vectors.npz, written by
tests/golden/make_moment_vectors.py): `moment_reduce` of
compute_statistical_moments.py for the zeroth, first and second orders over
(longitude, latitude) and over time, and compute_averages.py's
`v * get_lat_weights` reduced by sum / count.  The operators run on a NumPy
interpretation of the C ABI (tests/fake_ctx_average.py).  The zeroth order is
exact; the others are within the reference's own float32 or float64 pairwise
summation error plus this package's stated bound (DESIGN.md section 8g)."""
import math
import os

import numpy as np
import pytest

import fake_ctx_average
from weatherbench2_b200 import preprocessing as pp
from weatherbench2_b200 import xarray_lite as xl

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden',
                      'reference_moment_vectors.npz')
DIMS = ('time', 'level', 'longitude', 'latitude')


def _vectors():
  return np.load(GOLDEN)


def _dataset(x):
  return xl.Dataset({'t': (DIMS, x)}, {
      'time': np.arange(5), 'level': np.array([500.0, 850.0]),
      'longitude': np.arange(9) * 40.0,
      'latitude': np.linspace(-90.0, 90.0, 7)})


def _rtol(dtype, n):
  """The reference's pairwise-sum error plus this package's bound, relative
  (every field here is positive, so sum |x| / count is the mean)."""
  if dtype == np.float32:
    return (math.log2(n) + 3) * 2.0 ** -24
  return (math.log2(n) + math.ceil(n / 32) + 9) * 2.0 ** -53


@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('reduce_dims', [('longitude', 'latitude'), ('time',)])
def test_moment_reduce_matches_the_reference(dtype, reduce_dims):
  v = _vectors()
  x = v[f'{dtype}|x']
  key = f'{dtype}|{"_".join(reduce_dims)}'
  n = math.prod(x.shape[DIMS.index(d)] for d in reduce_dims)
  with fake_ctx_average.installed():
    for order in pp.MOMENT_ORDERS:
      got = pp.moment_reduce(_dataset(x), order, reduce_dims)['t'].values
      want = v[f'{key}|{order}']
      assert got.dtype == want.dtype and got.shape == want.shape, order
      np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
      if order == 'zeroth':
        np.testing.assert_array_equal(got, want)
      else:
        np.testing.assert_allclose(got, want, rtol=_rtol(x.dtype, n), atol=0,
                                   err_msg=order)


@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('avg', [('time', 'latitude'),
                                 ('longitude', 'latitude')])
@pytest.mark.parametrize('skipna', [False, True])
def test_compute_averages_matches_the_reference_weighting(dtype, avg, skipna):
  v = _vectors()
  x = v[f'{dtype}|x']
  n = math.prod(x.shape[DIMS.index(d)] for d in avg)
  with fake_ctx_average.installed():
    got = pp.compute_averages(_dataset(x), list(avg), skipna=skipna,
                              time_start=None, time_stop=None)['t'].values
  want = v[f'{dtype}|avg|{"_".join(avg)}|{"skipna" if skipna else "noskip"}']
  assert got.dtype == np.float64 and got.shape == want.shape
  np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
  np.testing.assert_allclose(got, want, atol=0,
                             rtol=_rtol(np.float64, n))

"""GPU tests of wb2_quantile / wb2_quantile_host (csrc/quantile.cu) and
preprocessing.compute_quantiles: every output bit-equal to
tests/quantile_oracle.py (np.quantile / np.nanquantile), NaN positions
included; the sign of a zero may differ only in cells that hold both +0 and
-0.  Each path is reached at the edges of its choice: n = 1, 2, 50, 63, 64
(register networks), 65, the largest staged n and the smallest unstaged one
(radix select), and 43,828; inner extents 1, 6, 31, 32, 33 and 721 x 1440;
both dtypes and both skipna; NaN fractions 0, 20 % and 100 % per cell, +-Inf,
constant and tied cells, +-0 and 1e5 + N(0, 1) data; 1, 7 and 128 quantiles.
Host input is streamed in many bands of both shapes."""
import math

import numpy as np
import pytest

import quantile_oracle as qo

pytestmark = pytest.mark.gpu

Q7 = [0.0, 1e-12, 1 / 3, 0.5, 0.999, 1 - 1e-12, 1.0]
# long-path tiles staged in shared memory up to these sample counts
# ((227 KB - 32 KB of histograms) / (33 x 4 B) and / (17 x 8 B))
STAGED_MAX = {np.float32: 1512, np.float64: 1468}


def _cells(nouter, n, ninner, dtype, seed):
  """[nouter][n][ninner] with a mix of cell kinds along the flat cell index:
  1e5 + N(0, 1), 20 % NaN, all NaN, +-Inf, constant, ties, +-0."""
  rs = np.random.RandomState(seed)
  x = (1e5 + rs.standard_normal((nouter, n, ninner))).astype(dtype)
  flat = x.transpose(0, 2, 1).reshape(-1, n)  # a copy: [cell][sample]
  kinds = np.arange(flat.shape[0]) % 9
  rows = [np.nonzero(kinds == k)[0] for k in range(9)]
  sub = flat[rows[1]]
  sub[rs.uniform(size=sub.shape) < 0.2] = np.nan
  flat[rows[1]] = sub
  flat[rows[2]] = np.nan
  sub = flat[rows[3]]
  u = rs.uniform(size=sub.shape)
  sub[u < 0.1] = np.inf
  sub[u > 0.9] = -np.inf
  flat[rows[3]] = sub
  flat[rows[4]] = dtype(2.5)
  flat[rows[5]] = np.round(rs.standard_normal((rows[5].size, n)) * 2)
  z = np.where(rs.uniform(size=(rows[6].size, n)) < 0.5, -0.0, 0.0)
  z[rs.uniform(size=z.shape) < 0.2] = 1.0
  flat[rows[6]] = z
  flat[rows[7]] = rs.standard_normal((rows[7].size, n)) * 1e-30
  if n > 2:
    flat[rows[8], 0] = np.nan  # one NaN: NaN without skipna, dropped with it
  return np.ascontiguousarray(
      flat.reshape(nouter, ninner, n).transpose(0, 2, 1))


def _mixed_zero(x, axis):
  z = x == 0
  return (z & np.signbit(x)).any(axis=axis) & (z & ~np.signbit(x)).any(axis=axis)


def _assert_bits(got, want, mixed, what):
  got, want = np.asarray(got), np.asarray(want)
  assert got.dtype == np.float64 and got.shape == want.shape, (
      what, got.dtype, got.shape, want.shape)
  np.testing.assert_array_equal(np.isnan(got), np.isnan(want), err_msg=what)
  same = (got.view(np.uint64) == want.view(np.uint64)) | np.isnan(want)
  same |= (want == 0) & (got == 0) & np.broadcast_to(mixed, want.shape)
  if not same.all():
    i = tuple(np.argwhere(~same)[0])
    raise AssertionError(f'{what}: {(~same).sum()} values differ, first at {i}: '
                         f'{got[i]!r} vs {want[i]!r}')


def _code(dtype):
  from weatherbench2_b200 import _lib
  return _lib.F32 if np.dtype(dtype) == np.float32 else _lib.F64


def _device(x, q, skipna):
  import torch
  from weatherbench2_b200 import _lib
  ctx = _lib.default_context()
  nouter, n, ninner = x.shape
  xd = torch.from_numpy(x).cuda()
  od = torch.full((len(q), nouter, ninner), 7.0, dtype=torch.float64,
                  device='cuda')
  ctx.quantile(xd.data_ptr(), _code(x.dtype), nouter, n, ninner, q, skipna,
               od.data_ptr())
  return od.cpu().numpy()


def _host(x, q, skipna, budget=1 << 30):
  from weatherbench2_b200 import _lib
  ctx = _lib.default_context()
  nouter, n, ninner = x.shape
  oh = np.full((len(q), nouter, ninner), 7.0)
  ctx.quantile_host(x.ctypes.data, _code(x.dtype), nouter, n, ninner, q,
                    skipna, budget, oh.ctypes.data)
  return oh


def _bands(x, nq, budget):
  """The band count of stream_series_bands (csrc/stage.cuh) for this call."""
  nouter, n, ninner = x.shape
  per_cell = n * x.dtype.itemsize + nq * 8
  cells = max(1, budget // (2 * per_cell))
  nb = min(cells, ninner)
  ko = max(1, min(cells // ninner, nouter)) if nb == ninner else 1
  return math.ceil(nouter / ko) * math.ceil(ninner / nb)


def _check(x, q, skipna, what, host=True):
  want = qo.quantile(x, q, skipna)
  mixed = _mixed_zero(x, 1)[None]
  _assert_bits(_device(x, q, skipna), want, mixed, f'{what} device')
  if host:
    _assert_bits(_host(x, q, skipna), want, mixed, f'{what} host')


@pytest.mark.parametrize('dtype', [np.float32, np.float64])
@pytest.mark.parametrize('n', [1, 2, 3, 50, 63, 64, 65, 'staged', 'unstaged'])
def test_every_path_at_its_edges(n, dtype):
  if n == 'staged':
    n = STAGED_MAX[dtype]
  elif n == 'unstaged':
    n = STAGED_MAX[dtype] + 1
  for ninner in (1, 6, 31, 32, 33):
    nouter = max(2, 300 // ninner) if n <= 64 else 3
    x = _cells(nouter, n, ninner, dtype, seed=n * 100 + ninner)
    for skipna in (False, True):
      _check(x, Q7, skipna, f'n={n} ninner={ninner} skipna={skipna}')


@pytest.mark.parametrize('dtype', [np.float32, np.float64])
def test_climatological_sample_count(dtype):
  # 30 years of 6-hourly samples per cell: the unstaged radix select
  x = _cells(1, 43828, 40, dtype, seed=43828)
  for skipna in (False, True):
    _check(x, [0.01, 0.5, 0.99], skipna, f'n=43828 skipna={skipna}')


@pytest.mark.parametrize('n', [5, 1460])
def test_full_grid(n):
  """721 x 1440 inner cells; n = 1460 on a seeded row band of the grid."""
  ninner = 721 * 1440 if n == 5 else 1440 * 3
  x = _cells(1, n, ninner, np.float32, seed=n)
  _check(x, [0.1, 0.5, 0.9], True, f'n={n} ninner={ninner}', host=(n == 5))


@pytest.mark.parametrize('n', [20, 65])
@pytest.mark.parametrize('nq', [1, 128])
def test_one_and_128_quantiles(n, nq):
  q = [0.3] if nq == 1 else list(np.linspace(0, 1, nq))
  q = q if nq == 1 else q[::-1]  # unsorted: no order is assumed
  x = _cells(4, n, 37, np.float64, seed=nq + n)
  for skipna in (False, True):
    _check(x, q, skipna, f'n={n} nq={nq}')


@pytest.mark.parametrize('shape', [(200, 70, 3), (3, 70, 5000), (2, 1500, 999)])
def test_host_streamed_in_bands(shape):
  """Whole outer rows per band, and parts of one outer index per band; band
  counts that do not divide the cells; the launch count is the band count."""
  from weatherbench2_b200 import _lib
  ctx = _lib.default_context()
  x = _cells(*shape, np.float32, seed=sum(shape))
  q = [0.0, 0.25, 0.999]
  per_cell = shape[1] * 4 + len(q) * 8
  cells = shape[0] * shape[2]
  budget = 2 * per_cell * (cells // 7 + (3 if shape[2] == 3 else 1))
  nb = _bands(x, len(q), budget)
  assert nb >= 5
  ctx.synchronize()
  before = ctx.launch_count
  got = _host(x, q, True, budget)
  ctx.synchronize()
  assert ctx.launch_count - before == nb
  _assert_bits(got, qo.quantile(x, q, True), _mixed_zero(x, 1)[None],
               f'bands {shape}')


@pytest.mark.parametrize('on_device', [True, False])
def test_operator_non_adjacent_dims(on_device):
  import torch
  from weatherbench2_b200 import preprocessing
  from weatherbench2_b200 import xarray_lite as xl
  rs = np.random.RandomState(5)
  x = (1e5 + rs.standard_normal((24, 7, 90))).astype(np.float32)
  x[3, 2, :5] = np.nan
  y = rs.standard_normal((24, 7)).astype(np.float64)
  data = torch.from_numpy(x).cuda() if on_device else x
  ds = xl.Dataset({'t': (('time', 'lat', 'lon'), data),
                   'u': (('time', 'lat'), torch.from_numpy(y).cuda()
                         if on_device else y)},
                  coords={'time': np.arange(24), 'lat': np.arange(7.0),
                          'lon': np.arange(90.0)})
  q = [0.1, 0.5, 0.9]
  for skipna in (False, True):
    got = preprocessing.compute_quantiles_core(ds, q, ['lon', 'time'],
                                               skipna=skipna, name_suffix='_q')
    t, u = got['t_q'], got['u_q']
    assert t.dims == ('quantile', 'lat') and u.dims == ('quantile', 'lat')
    assert xl._is_torch(t.data) == on_device  # pylint: disable=protected-access
    fn = np.nanquantile if skipna else np.quantile
    with np.errstate(invalid='ignore'):
      want_t = np.asarray(fn(x, q, axis=(0, 2)), np.float64)
    _assert_bits(t.values, want_t, False, f't skipna={skipna}')
    _assert_bits(u.values, np.quantile(y, q, axis=0), False, 'u')
    assert list(got.coords) == ['lat', 'quantile']


def test_every_argument_error_launches_nothing():
  import torch
  from weatherbench2_b200 import _lib
  ctx = _lib.default_context()
  x = torch.zeros((2, 100, 3), device='cuda')
  out = torch.empty((2, 2, 3), dtype=torch.float64, device='cuda')
  xh = np.zeros((2, 100, 3), np.float32)
  oh = np.empty((2, 2, 3))
  good = dict(x=x.data_ptr(), dtype=_lib.F32, nouter=2, nsample=100, ninner=3,
              quantiles=[0.25, 0.75], skipna=False, out=out.data_ptr())
  goodh = dict(good, x=xh.ctypes.data, out=oh.ctypes.data, budget=1 << 20)
  bad = [(dict(dtype=2), 'dtype'), (dict(dtype=-1), 'dtype'),
         (dict(nsample=0), 'nsample'), (dict(nsample=-5), 'nsample'),
         (dict(nouter=-1), 'nouter'), (dict(ninner=-1), 'ninner'),
         (dict(nquantile=0), 'nquantile'), (dict(nquantile=129), 'nquantile'),
         (dict(quantiles=None, nquantile=2), 'quantiles'),
         (dict(quantiles=[0.5, 1.5]), r'quantiles\[1\]'),
         (dict(quantiles=[-1e-300, 0.5]), r'quantiles\[0\]'),
         (dict(quantiles=[0.5, float('nan')]), r'quantiles\[1\]'),
         (dict(x=None), 'x is NULL'), (dict(out=None), 'out is NULL')]
  ctx.synchronize()
  before = ctx.launch_count
  for change, name in bad:
    with pytest.raises(_lib.Wb2Error, match=name):
      ctx.quantile(**dict(good, **change))
    with pytest.raises(_lib.Wb2Error, match=name):
      ctx.quantile_host(**dict(goodh, **change))
  ctx.synchronize()
  assert ctx.launch_count == before
  ctx.quantile(**dict(good, nouter=0))  # nothing to do
  ctx.quantile_host(**dict(goodh, ninner=0))
  ctx.quantile(**good)
  ctx.synchronize()
  assert ctx.launch_count - before == 1
  np.testing.assert_array_equal(out.cpu().numpy(), 0.0)

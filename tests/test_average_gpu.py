"""GPU tests of wb2_average / wb2_average_host (csrc/average.cu) and the
operators compute_averages, moment_reduce and compute_statistical_moments:
every output bit-equal to tests/average_oracle.py, which restates the
header's summation order.  Covered: the canonical layouts R, K R, R K, K R K,
R K R and K R K R K, both kernels (k2 below and from 32), three reduced runs
through the operators' transposed copy, weights in r0 and in r1, n from 1
past the 65536-sample chunk, one cell of 2^28 samples, both dtypes, both
skipna settings, NaN and +-Inf fields, a float32 square that overflows and a
721 x 1440 field.  The host entry is bit-equal to the device entry at several
budgets with the predicted launch count; repeated calls give the same bits;
every argument error is raised with nothing launched; CUDA and NumPy inputs
of the operators give the same bits."""
import numpy as np
import pandas as pd
import pytest

import average_oracle as ao
import wb2_testdata

pytestmark = pytest.mark.gpu

C = ao.CHUNK


def _field(shape, dtype, seed, special=True):
  rs = np.random.RandomState(seed)
  x = (rs.standard_normal(shape) * 10.0 ** rs.randint(-3, 4, size=shape))
  x = x.astype(dtype)
  if special:
    u = rs.uniform(size=shape)
    x[u < 0.05] = np.nan
    x[(u > 0.05) & (u < 0.053)] = np.inf
    x[(u > 0.053) & (u < 0.055)] = -np.inf
    x[(u > 0.055) & (u < 0.056)] = 3e20 if dtype == np.float32 else 1e160
    flat = x.reshape(-1)
    if flat.size > 40:
      flat[:7] = np.nan  # an all-NaN cell in most layouts
  return x


def _same(got, want, what):
  got, want = np.asarray(got), np.asarray(want)
  assert got.dtype == want.dtype and got.shape == want.shape, (
      what, got.dtype, want.dtype, got.shape, want.shape)
  nan = np.isnan(want)
  np.testing.assert_array_equal(np.isnan(got), nan, err_msg=what)
  u = np.uint32 if got.dtype == np.float32 else np.uint64
  same = (got.view(u) == want.view(u)) | nan
  if not same.all():
    i = tuple(np.argwhere(~same)[0])
    raise AssertionError(f'{what}: {(~same).sum()} values differ, first at '
                         f'{i}: {got[i]!r} vs {want[i]!r}')


def _device(x5, skipna, weights=None, wdiv=1):
  import torch
  from weatherbench2_b200 import _lib
  ctx = _lib.default_context()
  k0, _, k1, _, k2 = x5.shape
  xd = torch.from_numpy(np.ascontiguousarray(x5)).cuda()
  mt = torch.float64 if weights is not None else xd.dtype
  outs = [torch.empty((k0, k1, k2), dtype=t, device='cuda')
          for t in (mt, mt, torch.float64)]
  ctx.average(xd.data_ptr(), _lib.F64 if x5.dtype == np.float64 else _lib.F32,
              x5.shape, skipna, *(o.data_ptr() for o in outs),
              weights=weights, wdiv=wdiv)
  torch.cuda.synchronize()
  return [o.cpu().numpy() for o in outs]


def _host(x5, skipna, budget, weights=None, wdiv=1):
  from weatherbench2_b200 import _lib
  ctx = _lib.default_context()
  k0, _, k1, _, k2 = x5.shape
  mt = np.float64 if weights is not None else x5.dtype
  outs = [np.full((k0, k1, k2), 7.0, t) for t in (mt, mt, np.float64)]
  x5 = np.ascontiguousarray(x5)
  ctx.average_host(x5.ctypes.data,
                   _lib.F64 if x5.dtype == np.float64 else _lib.F32, x5.shape,
                   skipna, budget, *(o.ctypes.data for o in outs),
                   weights=weights, wdiv=wdiv)
  return outs


LAYOUTS = {
    'R': (1, 3000, 1, 1, 1),
    'K R': (37, 1500, 1, 1, 1),
    'R K': (1, 70, 1, 1, 333),
    'R K narrow': (1, 70, 1, 1, 5),
    'K R K': (3, 40, 1, 1, 65),
    'R K R': (1, 9, 13, 200, 1),
    'K R K R K': (2, 5, 3, 7, 33),
    'K R K R k': (2, 5, 3, 70, 4),
}


@pytest.mark.parametrize('layout', list(LAYOUTS))
@pytest.mark.parametrize('dtype', [np.float32, np.float64])
@pytest.mark.parametrize('skipna', [False, True])
def test_layouts_bit_equal(layout, dtype, skipna):
  shape = LAYOUTS[layout]
  x5 = _field(shape, dtype, list(LAYOUTS).index(layout) * 2 + skipna)
  want = ao.canonical(x5, skipna)
  for got in (_device(x5, skipna), _host(x5, skipna, 1 << 26),
              _host(x5, skipna, 3 * (x5.nbytes // shape[0] // shape[2]))):
    for g, w, name in zip(got, want, ('mean', 'mean_sq', 'frac')):
      _same(g, w, f'{layout} {name}')


@pytest.mark.parametrize('where', ['r0', 'r1'])
@pytest.mark.parametrize('dtype', [np.float32, np.float64])
@pytest.mark.parametrize('skipna', [False, True])
def test_weights_in_r0_and_r1(where, dtype, skipna):
  for shape in ((2, 5, 3, 7, 33), (4, 19, 6, 36, 1)):
    x5 = _field(shape, dtype, 11)
    rs = np.random.RandomState(2)
    if where == 'r0':
      w, wdiv = rs.uniform(0.1, 2.0, size=shape[1]), shape[3]
    else:
      w, wdiv = rs.uniform(0.1, 2.0, size=shape[3]), 1
    want = ao.canonical(x5, skipna, w, wdiv)
    for got in (_device(x5, skipna, w, wdiv),
                _host(x5, skipna, 1 << 24, w, wdiv)):
      for g, ww in zip(got, want):
        _same(g, ww, f'{shape} weights in {where}')


@pytest.mark.parametrize('n', [1, 2, 31, 32, 33, 1000, C - 1, C, C + 1,
                               2 * C + 5])
@pytest.mark.parametrize('kernel', ['warp', 'cell'])
def test_sample_counts_across_the_chunk(n, kernel):
  shape = (3, n, 1, 1, 1) if kernel == 'warp' else (1, n, 1, 1, 40)
  for dtype, skipna in ((np.float32, True), (np.float64, False)):
    x5 = _field(shape, dtype, n % 977, special=n > 2)
    want = ao.canonical(x5, skipna)
    got = _device(x5, skipna)
    for g, w in zip(got, want):
      _same(g, w, f'n={n} {kernel}')


def test_one_cell_of_2_28_samples():
  import torch
  from weatherbench2_b200 import _lib
  ctx = _lib.default_context()
  n = 1 << 28
  g = torch.Generator(device='cuda').manual_seed(4)
  ints = torch.randint(0, 8, (n,), device='cuda', generator=g,
                       dtype=torch.int64)
  x = ints.to(torch.float32)
  x[12345] = float('nan')
  ints[12345] = 0
  # small integers: every partial sum is exact, whatever the order
  s1 = int(ints.sum())
  s2 = int((ints * ints).sum())
  outs = [torch.empty(1, dtype=t, device='cuda')
          for t in (torch.float32, torch.float32, torch.float64)]
  for skipna in (True, False):
    ctx.average(x.data_ptr(), _lib.F32, (1, n, 1, 1, 1), skipna,
                *(o.data_ptr() for o in outs))
    m, q, fr = (o.item() for o in outs)
    assert fr == (n - 1) / n
    if skipna:
      assert m == float(np.float32(s1 / (n - 1)))
      assert q == float(np.float32(s2 / (n - 1)))
    else:
      assert np.isnan(m) and np.isnan(q)
  del x, ints


def test_full_size_field():
  # a global latitude-weighted mean per step (K R) and a time-mean map (R K)
  lat = np.linspace(-90, 90, 721)
  from weatherbench2_b200 import _spatial as sp
  w = sp.lat_weights(lat)
  x = _field((3, 721, 1440), np.float32, 21)
  want = ao.canonical(x.reshape(3, 721 * 1440, 1, 1, 1), True, w, 1440)
  got = _device(x.reshape(3, 721 * 1440, 1, 1, 1), True, w, 1440)
  for g, ww in zip(got, want):
    _same(g, ww, 'global mean')
  x5 = x.reshape(1, 3, 1, 1, 721 * 1440)
  want = ao.canonical(x5, False)
  for got in (_device(x5, False), _host(x5, False, 1 << 26)):
    for g, ww in zip(got, want):
      _same(g, ww, 'time-mean map')


def test_host_bands_and_launch_count():
  from weatherbench2_b200 import _lib
  ctx = _lib.default_context()
  shape = (3, 50, 7, 40, 1)
  x5 = _field(shape, np.float32, 5)
  want = ao.canonical(x5, True)
  dev = _device(x5, True)
  # one k1 slice: 2000 float32 samples and three outputs, in both buffers
  slice_cost = 2 * (2000 * 4 + 4 + 4 + 8)
  for budget, bands in ((slice_cost, 21), (3 * slice_cost, 9),
                        (14 * slice_cost, 2), (1 << 30, 1)):
    before = ctx.launch_count
    got = _host(x5, True, budget)
    assert ctx.launch_count - before == bands, budget
    for g, d, w in zip(got, dev, want):
      _same(g, w, f'budget {budget}')
      _same(g, d, f'budget {budget} vs device')
  with pytest.raises(_lib.Wb2Error, match='budget'):
    _host(x5, True, slice_cost - 1)
  # n past one chunk: three launches per band
  x5 = _field((2, C + 3, 3, 1, 1), np.float32, 6)
  before = ctx.launch_count
  got = _host(x5, False, 1 << 30)
  assert ctx.launch_count - before == 3
  for g, w in zip(got, ao.canonical(x5, False)):
    _same(g, w, 'chunked host')


@pytest.mark.parametrize('layout,shape', [
    ('R K', (1, 37, 1, 1, 5000)),
    ('K R K R K', (2, 9, 3, 11, 700)),
    ('K R K R K weighted', (2, 9, 3, 11, 700))])
def test_host_streams_cells_of_a_k1_slice_larger_than_the_budget(layout,
                                                                shape):
  """Bands split k2 on whole cells when one k1 slice exceeds the budget."""
  from weatherbench2_b200 import _lib
  ctx = _lib.default_context()
  k0, r0, k1, r1, k2 = shape
  n = r0 * r1
  w, wdiv = None, 1
  if layout.endswith('weighted'):
    w, wdiv = np.random.RandomState(3).uniform(0.1, 2.0, size=r0), r1
  x5 = _field(shape, np.float32, 17)
  dev = _device(x5, True, w, wdiv)
  ob = 8 if w is not None else 4
  cell_cost = 2 * (n * 4 + ob + ob + 8)
  slice_cost = k2 * cell_cost
  for cells in (1, 7, 333, k2 - 1):
    budget = cells * cell_cost
    assert budget < slice_cost
    before = ctx.launch_count
    got = _host(x5, True, budget, w, wdiv)
    assert ctx.launch_count - before == k0 * k1 * -(-k2 // cells), cells
    for g, d in zip(got, dev):
      _same(g, d, f'{layout} {cells} cells per band')
  for g, ww in zip(got, ao.canonical(x5, True, w, wdiv)):
    _same(g, ww, f'{layout} oracle')
  with pytest.raises(_lib.Wb2Error, match='budget of'):
    _host(x5, True, cell_cost - 1, w, wdiv)


def test_time_mean_map_streamed_in_many_bands():
  """A NumPy time-mean map bigger than the operators' staging budget."""
  from weatherbench2_b200 import _lib
  from weatherbench2_b200 import preprocessing as pp
  from weatherbench2_b200 import xarray_lite as xl
  ctx = _lib.default_context()
  x = _field((200, 721, 1440), np.float32, 19)  # 0.83 GB
  ds = xl.Dataset({'t': (('time', 'latitude', 'longitude'), x)},
                  {'time': pd.date_range('2020-01-01', periods=200).values})
  saved = pp.AVERAGE_STREAM_BUDGET_BYTES
  pp.AVERAGE_STREAM_BUDGET_BYTES = 1 << 28
  try:
    before = ctx.launch_count
    out = _both(lambda z: pp.compute_averages(z, ['time']), ds)
    assert ctx.launch_count - before > 4  # the NumPy call took several bands
  finally:
    pp.AVERAGE_STREAM_BUDGET_BYTES = saved
  want = ao.canonical(x.reshape(1, 200, 1, 1, 721 * 1440), False)[0]
  _same(out['t'].values, want.reshape(721, 1440), 'time-mean map')


def test_repeated_calls_give_the_same_bits():
  x5 = _field((1, 5 * C + 11, 1, 1, 1), np.float32, 8, special=False)
  a = _device(x5, False)
  b = _device(x5, False)
  for u, v in zip(a, b):
    _same(u, v, 'repeat')


def test_argument_errors():
  import torch
  from weatherbench2_b200 import _lib
  ctx = _lib.default_context()
  x = torch.zeros(24, device='cuda')
  o = torch.full((6,), 5.0, device='cuda')
  good = dict(x=x.data_ptr(), dtype=_lib.F32, shape=(2, 4, 3, 1, 1),
              skipna=False, mean=o.data_ptr())
  w = np.ones(3)
  before = ctx.launch_count
  for change, name in ((dict(dtype=5), 'dtype'),
                       (dict(shape=(2, 0, 3, 1, 1)), 'r0 and r1'),
                       (dict(shape=(2, 4, 3, 0, 1)), 'r0 and r1'),
                       (dict(shape=(2, 4, -3, 1, 1)), 'kept extents'),
                       (dict(weights=w), 'weights'),
                       (dict(weights=np.ones(2), wdiv=3), 'weights'),
                       (dict(mean=0), 'no output'),
                       (dict(x=0), 'x is NULL')):
    with pytest.raises(_lib.Wb2Error, match=name):
      ctx.average(**dict(good, **change))
    with pytest.raises(_lib.Wb2Error, match=name):
      ctx.average_host(**dict(good, budget=1 << 20, **change))
  assert ctx.launch_count == before
  ctx.average(**dict(good, shape=(2, 4, 0, 1, 1)))  # no cells: a no-op
  assert ctx.launch_count == before
  assert (o.cpu() == 5.0).all()


# -- the operators on CUDA and NumPy input --------------------------------------
def _both(fn, ds_np):
  """fn on the NumPy dataset and on the same dataset with CUDA tensors."""
  import torch
  from weatherbench2_b200 import xarray_lite as xl
  ds_cu = xl.Dataset({k: (v.dims, torch.from_numpy(v.values).cuda())
                      for k, v in ds_np.items()}, ds_np.coords)
  a, b = fn(ds_np), fn(ds_cu)
  assert list(a.keys()) == list(b.keys())
  for k in a.keys():
    assert a[k].dims == b[k].dims
    assert b[k].data.is_cuda and isinstance(a[k].data, np.ndarray)
    _same(b[k].data.cpu().numpy(), a[k].values, k)
  return a


def _forecast():
  from weatherbench2_b200 import xarray_lite as xl
  d = wb2_testdata.random_like(wb2_testdata.mock_forecast_data(
      ensemble_size=3, variables_3d=('geopotential', 'temperature'),
      variables_2d=(), time_start='2020-05-25', time_stop='2020-07-10'))
  return xl.Dataset(d['vars'], d['coords']), d


def test_reference_cases_cuda_and_numpy():
  from weatherbench2_b200 import metrics
  from weatherbench2_b200 import preprocessing as pp
  ds, d = _forecast()
  t = pd.DatetimeIndex(d['coords']['time'])
  sel = (t >= '2020-06-01') & (t <= '2020-07-01')
  kw = dict(variables=['geopotential', 'temperature'],
            time_start='2020-06-01', time_stop='2020-07-01')
  out = _both(lambda z: pp.compute_averages(z, ['time', 'longitude'],
                                            levels=[700], **kw), ds)
  for name in out.keys():
    x = d['vars'][name][1][:, :, sel][:, :, :, [1]]
    np.testing.assert_allclose(out[name].values, x.mean(axis=(2, 4)),
                               rtol=1e-5, atol=1e-8)
  out = _both(lambda z: pp.compute_averages(z, ['time', 'latitude'], **kw), ds)
  w = metrics.get_lat_weights(ds).values
  for name in out.keys():
    tm = d['vars'][name][1][:, :, sel].mean(axis=2)
    np.testing.assert_allclose(out[name].values,
                               (tm * w).sum(axis=-1) / w.sum(),
                               rtol=1e-5, atol=1e-8)


@pytest.mark.parametrize('dtype', [np.float32, np.float64])
def test_operators_cuda_and_numpy(dtype):
  from weatherbench2_b200 import preprocessing as pp
  from weatherbench2_b200 import xarray_lite as xl
  x = _field((6, 3, 19, 36), dtype, 13)
  ds = xl.Dataset(
      {'t': (('time', 'level', 'latitude', 'longitude'), x)},
      {'time': pd.date_range('2019-12-29', periods=6).values,
       'level': np.array([500.0, 700.0, 850.0]),
       'latitude': np.linspace(-90, 90, 19),
       'longitude': np.arange(36) * 10.0})
  for dims in (['time', 'longitude'], ['time', 'latitude'], ['level'],
               ['time', 'latitude', 'longitude'],
               ['time', 'level', 'latitude', 'longitude']):
    for skipna in (False, True):
      _both(lambda z: pp.compute_averages(z, dims, skipna=skipna,
                                          time_start=None), ds)
  # three reduced runs: one transposed copy
  x5 = _field((3, 4, 19, 6, 7), dtype, 14)
  ds5 = xl.Dataset({'v': (('a', 'b', 'latitude', 'd', 'e'), x5)},
                   {'latitude': np.linspace(-90, 90, 19)})
  out = _both(lambda z: pp.compute_averages(z, ['a', 'latitude', 'e']), ds5)
  from weatherbench2_b200 import metrics
  w = metrics.get_lat_weights(ds5).values
  _same(out['v'].values, ao.average(x5, [0, 2, 4], False, w, 2)[0], 'copy')
  for order in pp.MOMENT_ORDERS:
    _both(lambda z: pp.moment_reduce(z, order), ds)
  out = _both(lambda z: pp.compute_statistical_moments(
      z, start_year=2020, end_year=2020), ds)
  assert list(out.keys()) == ['t_zeroth', 't_first', 't_second']
  m, q, fr = ao.average(x[3:], [2, 3], skipna=True)
  for name, s in (('t_zeroth', fr), ('t_first', m), ('t_second', q)):
    assert out[name].dims == ('moment', 'level')
    _same(out[name].values[0], ao.average(s, [0], skipna=True)[0], name)

"""CPU tests of the quantiles of scripts/compute_quantiles.py: the header's
six-step contract (include/wb2b200.h) restated in tests/quantile_oracle.py and
held bit-equal to np.quantile / np.nanquantile on seeded cells; hand cases;
the reference test's case (compute_quantiles_test.py:65-139); and
preprocessing.compute_quantiles end to end on a NumPy interpretation of the
entries (tests/fake_ctx_quantile.py), with every error it raises."""
import numpy as np
import pandas as pd
import pytest

import fake_ctx_quantile
import quantile_oracle as qo
from weatherbench2_b200 import _lib
from weatherbench2_b200 import preprocessing as pp
from weatherbench2_b200 import xarray_lite as xl

Q = [0.0, 1e-12, 0.1, 0.25, 1 / 3, 0.5, 0.75, 0.9, 0.999, 1 - 1e-12, 1.0]


def _seeded_cell(rs, n, dtype):
  kind = rs.randint(6)
  if kind == 0:
    x = 1e5 + rs.standard_normal(n)
  elif kind == 1:
    x = np.round(rs.standard_normal(n) * 2)  # ties
  elif kind == 2:
    x = rs.choice([-0.0, 0.0, 1.0, -1.0], size=n)
  else:
    x = rs.standard_normal(n) * 10.0 ** rs.randint(-30, 30)
  x = x.astype(dtype)
  for v, p in ((np.nan, 0.15), (np.inf, 0.05), (-np.inf, 0.05)):
    if rs.uniform() < 0.4:
      x[rs.uniform(size=n) < p] = v
  if rs.uniform() < 0.03:
    x[:] = np.nan
  return x


def _same_bits(a, b, cell=None):
  """Bit equality, NaN payloads aside; with `cell`, the sign of a zero may
  differ when the cell holds both +0 and -0 (their order is undefined in
  numpy's partition as in the kernels)."""
  a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
  same = (a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))
  if cell is not None:
    z = cell == 0
    if (z & np.signbit(cell)).any() and (z & ~np.signbit(cell)).any():
      same |= (a == 0) & (b == 0)
  return bool(same.all())


@pytest.mark.parametrize('dtype', [np.float32, np.float64])
@pytest.mark.parametrize('n', [1, 2, 3, 5, 64, 65, 1461])
@pytest.mark.parametrize('skipna', [False, True])
def test_contract_is_numpy_bit_for_bit(n, dtype, skipna):
  rs = np.random.RandomState(n * 7 + int(skipna) + (dtype == np.float64) * 3)
  for _ in range(60 if n < 1000 else 12):
    x = _seeded_cell(rs, n, dtype)
    want = qo.quantile(x[None, :, None], Q, skipna)[:, 0, 0]
    got = qo.contract(x, Q, skipna)
    assert _same_bits(got, want, x), (x, got, want)


def test_hand_cases():
  c = qo.contract
  assert c(np.float64([1, 2, 3, 4]), [0.5])[0] == 2.5
  np.testing.assert_array_equal(c(np.float64([4, 1, 3, 2]), [0, 1]), [1, 4])
  np.testing.assert_array_equal(c(np.float32([7]), [0, 0.3, 1]), [7, 7, 7])
  assert np.isnan(c(np.float64([np.nan] * 3), [0.5], True)).all()
  assert np.isnan(c(np.float64([1, np.nan, 3]), [0.5], False)).all()
  assert c(np.float64([1, np.nan, 3]), [0.5], True)[0] == 2.0
  assert np.isnan(c(np.float64([np.inf]), [0, 0.5, 1])).all()
  r = c(np.float64([1, np.inf]), [0, 0.25, 1])
  assert np.isnan(r[0]) and r[1] == np.inf and np.isnan(r[2])
  np.testing.assert_array_equal(c(np.float32([1, 16777218]), [0.5, 0.25]),
                                [8388610, 4194305])
  np.testing.assert_array_equal(c(np.float64([1, 16777218]), [0.5, 0.25]),
                                [8388609.5, 4194305.25])
  for x, q in (([1, 2, 3, 4], [0.5]), ([1, np.inf], [0, 0.25, 1]),
               ([np.inf], [0.5])):
    for dt in (np.float32, np.float64):
      a = np.asarray(x, dt)
      assert _same_bits(c(a, q), qo.quantile(a[None, :, None], q)[:, 0, 0])


def _reference_case():
  times = pd.DatetimeIndex(['2023-01-01', '2023-01-02', '2023-01-03',
                            '2023-01-04'])
  precip = np.random.RandomState(802701).rand(4, 50, 6)
  coords = {'time': times.values, 'lat': np.arange(50),
            'timedelta': np.arange(6)}
  dims = ('time', 'lat', 'timedelta')
  return xl.Dataset({'precip': (dims, precip),
                     'should_drop': (dims, precip * 2)}, coords), precip


def test_reference_case():
  ds, precip = _reference_case()
  with fake_ctx_quantile.installed() as fake:
    out = pp.compute_quantiles(ds, [0.2, 0.8], 'lat', variables=['precip'],
                               time_start='2023-01-01',
                               time_stop='2023-01-03',
                               name_suffix='_quantile')
  assert set(out.dims) == {'time', 'timedelta', 'quantile'}
  assert list(out.keys()) == ['precip_quantile']
  da = out['precip_quantile']
  assert da.dims == ('quantile', 'time', 'timedelta')
  want = np.quantile(precip[:3], [0.2, 0.8], axis=1)
  np.testing.assert_array_equal(da.values, want)
  assert out.coords['quantile'].values.dtype == np.float64
  np.testing.assert_array_equal(out.coords['quantile'].values, [0.2, 0.8])
  assert 'lat' not in out.coords and out.sizes['time'] == 3
  assert fake.calls == [('quantile_host', 3, 50, 6, 2, False,
                         pp.QUANTILE_STREAM_BUDGET_BYTES)]


def _dataset(dtype=np.float32):
  rs = np.random.RandomState(3)
  x = rs.standard_normal((5, 4, 3, 6)).astype(dtype)
  x[1, 2, 0, :2] = np.nan
  coords = {'time': pd.date_range('2020-01-01', periods=5).values,
            'level': np.array([500.0, 700.0, 850.0, 1000.0]),
            'lat': np.arange(3.0), 'lon': np.arange(6.0) * 60,
            'land': (('lat', 'lon'), rs.uniform(size=(3, 6)))}
  dims = ('time', 'level', 'lat', 'lon')
  return xl.Dataset({'t': (dims, x, {'units': 'K'}),
                     'z': (('lat', 'lon'), rs.standard_normal((3, 6)),
                           {'units': 'm'})}, coords, {'title': 'x'}), x


@pytest.mark.parametrize('dim,axes', [
    (['time', 'lat'], (0, 2)), (['lon', 'level'], (1, 3)),
    (['time', 'level', 'lat', 'lon'], (0, 1, 2, 3)), ('level', (1,)),
    (['lat', 'lon'], (2, 3))])
@pytest.mark.parametrize('skipna', [False, True])
def test_operator_layouts(dim, axes, skipna):
  ds, x = _dataset()
  q = [0.1, 0.5, 0.95]
  with fake_ctx_quantile.installed() as fake:
    out = pp.compute_quantiles_core(ds, q, dim, skipna=skipna)
  dims = [dim] if isinstance(dim, str) else dim
  keep = tuple(d for d in ('time', 'level', 'lat', 'lon') if d not in dims)
  t = out['t']
  assert t.dims == ('quantile',) + keep and t.attrs == {} and out.attrs == {}
  with np.errstate(invalid='ignore'):
    fn = np.nanquantile if skipna else np.quantile
    want = np.asarray(fn(x, q, axis=axes), np.float64)
  np.testing.assert_array_equal(t.values, want)
  # a variable without the reduced dims passes through with its attrs
  if not {'lat', 'lon'} & set(dims):
    assert out['z'].dims == ('lat', 'lon') and out['z'].attrs == {'units': 'm'}
  else:
    assert out['z'].dims[0] == 'quantile'
  # coordinates along reduced dims are dropped, the others kept
  for name in ('time', 'level', 'lat', 'lon'):
    assert (name in out.coords) == (name not in dims)
  assert ('land' in out.coords) == (not {'lat', 'lon'} & set(dims))
  # adjacent reduced dims are read in place, others after one transpose:
  # either way the entry sees [outer][n][inner]
  (_, nouter, n, ninner, nq, _, _) = fake.calls[0]
  assert n == int(np.prod([x.shape[a] for a in axes])) and nq == 3
  if axes == (1,):
    assert (nouter, ninner) == (5, 18)
  elif axes == (0, 2):
    assert (nouter, ninner) == (1, 24)


def test_selection():
  ds, x = _dataset()
  with fake_ctx_quantile.installed():
    out = pp.compute_quantiles(ds, [0.5], 'time', variables=['t'],
                               levels=['850', 500], time_start='2020-01-02',
                               time_stop='2020-01-04')
  assert list(out.keys()) == ['t']
  np.testing.assert_array_equal(out.coords['level'].values, [850.0, 500.0])
  want = np.quantile(x[1:4][:, [2, 0]], [0.5], axis=0)
  np.testing.assert_array_equal(out['t'].values, want)
  with fake_ctx_quantile.installed():
    out = pp.compute_quantiles(ds, [0.5], 'time')  # the script's 2020 range
    np.testing.assert_array_equal(out['t'].values,
                                  np.quantile(x, [0.5], axis=0))
    with pytest.raises(ValueError, match='empty'):
      pp.compute_quantiles(ds, [0.5], 'time', time_start='2021-01-01')
    out = pp.compute_quantiles(ds, [0.5], 'lat', time_start='2021-01-01')
  assert out['t'].shape == (1, 0, 4, 6)


def test_errors():
  ds, _ = _dataset()
  with fake_ctx_quantile.installed() as fake:
    for q in ([1.5], [-0.1], [0.5, float('nan')]):
      with pytest.raises(ValueError, match=r'Expected all quantiles to be in'):
        pp.compute_quantiles_core(ds, q, 'time')
    with pytest.raises(ValueError, match='128'):
      pp.compute_quantiles_core(ds, list(np.linspace(0, 1, 129)), 'time')
    with pytest.raises(ValueError, match='nope'):
      pp.compute_quantiles_core(ds, [0.5], ['time', 'nope'])
    bad = xl.Dataset({'i': (('time',), np.arange(4))})
    with pytest.raises(TypeError, match="'i'"):
      pp.compute_quantiles_core(bad, [0.5], 'time')
    empty = xl.Dataset({'e': (('time', 'x'), np.zeros((0, 3), np.float32))})
    with pytest.raises(ValueError, match='empty'):
      pp.compute_quantiles_core(empty, [0.5], 'time')
    assert not fake.calls
    # the entries' own checks
    ctx = _lib.default_context()
    x = np.zeros((2, 4, 3), np.float32)
    o = np.zeros((2, 2, 3))
    good = dict(x=x.ctypes.data, dtype=_lib.F32, nouter=2, nsample=4,
                ninner=3, quantiles=[0.1, 0.9], skipna=False, out=o.ctypes.data)
    for change, name in ((dict(dtype=5), 'dtype'), (dict(nsample=0), 'nsample'),
                         (dict(nquantile=129), 'nquantile'),
                         (dict(quantiles=[0.1, 2.0]), r'quantiles\[1\]')):
      with pytest.raises(_lib.Wb2Error, match=name):
        ctx.quantile(**dict(good, **change))
      with pytest.raises(_lib.Wb2Error, match=name):
        ctx.quantile_host(**dict(good, budget=1 << 20, **change))


def test_float64_and_other_array_types():
  ds, x = _dataset(np.float64)
  with fake_ctx_quantile.installed():
    out = pp.compute_quantiles_core(ds, [0.3], ['time'])
    lst = xl.Dataset({'a': (('s', 'c'), np.arange(12.0).reshape(4, 3))})
    got = pp.compute_quantiles_core(lst, [0.5], 's')
  np.testing.assert_array_equal(out['t'].values,
                                np.quantile(x, [0.3], axis=0))
  assert out['t'].values.dtype == np.float64
  np.testing.assert_array_equal(got['a'].values, [[4.5, 5.5, 6.5]])

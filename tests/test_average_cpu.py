"""CPU tests of the averages and raw moments of scripts/compute_averages.py and
compute_statistical_moments.py: the header's summation recipe restated in
tests/average_oracle.py and held to math.fsum within the stated bound; hand
cases of the NaN, Inf, count and overflow rules; the two cases of the
reference's compute_averages_test.py; and the three operators end to end on a
NumPy interpretation of the entries (tests/fake_ctx_average.py), with every
error they raise."""
import math
import os

import numpy as np
import pandas as pd
import pytest

import average_oracle as ao
import fake_ctx_average
import wb2_testdata
from weatherbench2_b200 import _lib
from weatherbench2_b200 import metrics
from weatherbench2_b200 import preprocessing as pp
from weatherbench2_b200 import xarray_lite as xl

HERE = os.path.dirname(os.path.abspath(__file__))


def _bits_equal(a, b):
  a, b = np.asarray(a), np.asarray(b)
  assert a.dtype == b.dtype and a.shape == b.shape
  same = (a == b) | (np.isnan(a) & np.isnan(b))
  same &= (np.signbit(a) == np.signbit(b)) | np.isnan(a)
  return bool(same.all())


@pytest.mark.parametrize('n', [1, 31, 32, 33, 1000, ao.CHUNK - 1, ao.CHUNK,
                               ao.CHUNK + 1, 3 * ao.CHUNK + 17])
def test_ordered_sum_within_the_header_bound(n):
  rs = np.random.RandomState(n % 1000)
  y = rs.standard_normal((3, n)) * 10.0 ** rs.randint(-5, 5, size=(3, n))
  y[1] = np.abs(y[1])
  got = ao.ordered_sum(y)
  for r in range(3):
    exact = math.fsum(y[r])
    bound = (math.ceil(n / 32) + 7) * 2.0 ** -53 * math.fsum(np.abs(y[r]))
    assert abs(got[r] - exact) <= bound * (1 + 1e-9), (n, r)


def test_ordered_sum_is_the_stated_order():
  # 2^53 + 1 - 2^53 depends on the order: class 0 gets 2^53 then 1, class 1
  # gets -2^53; the butterfly adds classes 0 + 16, ..., 0 + 1 last
  y = np.zeros((1, 64))
  y[0, 0], y[0, 32], y[0, 1] = 2.0 ** 53, 1.0, -2.0 ** 53
  assert ao.ordered_sum(y)[0] == 0.0  # (2^53 + 1) rounds to 2^53 first
  # chunk partials 2^53, 1, -2^53 added in chunk order: 1 is lost
  y = np.zeros((1, 2 * ao.CHUNK + 1))
  y[0, 0], y[0, ao.CHUNK], y[0, 2 * ao.CHUNK] = 2.0 ** 53, 1.0, -2.0 ** 53
  assert ao.ordered_sum(y)[0] == 0.0


def test_hand_cases():
  f64 = np.float64
  # count versus sum of weights, on a weighted field with NaN
  x = np.array([[1.0, np.nan, 3.0]])
  w = np.array([0.5, 1.0, 2.0])
  s1, _, cnt = ao.cell_stats(x, True, w)
  mean = ao.finish(s1, s1, cnt, 3, True, f64)[0]
  assert mean[0] == (0.5 + 6.0) / 2  # divided by the count 2, not 2.5
  assert mean[0] != (0.5 + 6.0) / 2.5
  # all-NaN cells: NaN with and without skipna, frac 0
  for skipna in (False, True):
    m, q, fr = ao.finish(*ao.cell_stats(np.full((1, 4), np.nan), skipna), 4,
                         skipna, f64)
    assert np.isnan(m[0]) and np.isnan(q[0]) and fr[0] == 0.0
  # Inf
  m, q, _ = ao.finish(*ao.cell_stats(np.array([[1.0, np.inf]]), False), 2,
                      False, f64)
  assert m[0] == np.inf and q[0] == np.inf
  m, q, _ = ao.finish(*ao.cell_stats(np.array([[np.inf, -np.inf]]), False), 2,
                      False, f64)
  assert np.isnan(m[0]) and q[0] == np.inf
  # a float32 square that overflows (np.square in float32), the mean not
  x = np.array([[3e20, 1.0]], np.float32)
  m, q, _ = ao.finish(*ao.cell_stats(x, False), 2, False, np.float32)
  assert m.dtype == np.float32 and m[0] == np.float32(1.5e20)
  assert q[0] == np.inf
  assert np.isfinite(np.float64(3e20) ** 2)
  # frac with and without NaN; skipna 0 propagates NaN into the mean only
  x = np.array([[1.0, 2.0, np.nan, 4.0], [1.0, 2.0, 3.0, 4.0]])
  m, _, fr = ao.finish(*ao.cell_stats(x, False), 4, False, f64)
  np.testing.assert_array_equal(fr, [0.75, 1.0])
  assert np.isnan(m[0]) and m[1] == 2.5
  m, _, _ = ao.finish(*ao.cell_stats(x, True), 4, True, f64)
  np.testing.assert_array_equal(m, [7 / 3, 2.5])


# -- the reference's scripts/compute_averages_test.py ---------------------------
def _forecast():
  """compute_averages_test's input: random_like(mock_forecast_data(
  ensemble_size=3)) plus the 'extra' variable, with a shorter time axis
  around the selected June 2020 window."""
  d = wb2_testdata.random_like(wb2_testdata.mock_forecast_data(
      ensemble_size=3, variables_3d=('geopotential', 'temperature'),
      variables_2d=('2m_temperature',), time_start='2020-05-25',
      time_stop='2020-07-10'))
  dims, t2 = d['vars']['2m_temperature']
  d['vars']['extra'] = (('extra_dim',) + dims, t2[None])
  coords = dict(d['coords'], extra_dim=np.array([1]))
  return xl.Dataset(d['vars'], coords), d


def _june(d):
  t = pd.DatetimeIndex(d['coords']['time'])
  return (t >= '2020-06-01') & (t <= '2020-07-01')


def test_reference_case_time_longitude():
  ds, d = _forecast()
  with fake_ctx_average.installed():
    out = pp.compute_averages(ds, ['time', 'longitude'], levels=[700],
                              variables=['geopotential', 'temperature'],
                              time_start='2020-06-01', time_stop='2020-07-01')
  assert list(out.keys()) == ['geopotential', 'temperature']
  sel = _june(d)
  lvl = list(d['coords']['level']).index(700)
  for name in out.keys():
    dims, x = d['vars'][name]
    x = x[:, :, sel][:, :, :, [lvl]]
    want = x.mean(axis=(2, 4))  # xarray's .mean(['time', 'longitude'])
    got = out[name]
    assert got.dims == ('realization', 'prediction_timedelta', 'level',
                        'latitude')
    np.testing.assert_allclose(got.values, want, rtol=1e-5, atol=1e-8)
  np.testing.assert_array_equal(out.coords['level'].values, [700.0])
  assert 'time' not in out.coords and 'longitude' not in out.coords


def test_reference_case_time_latitude_weighted():
  ds, d = _forecast()
  with fake_ctx_average.installed() as fake:
    out = pp.compute_averages(ds, ['time', 'latitude'],
                              variables=['geopotential', 'temperature'],
                              time_start='2020-06-01', time_stop='2020-07-01')
  sel = _june(d)
  w = metrics.get_lat_weights(ds).values
  for name in out.keys():
    _, x = d['vars'][name]
    tm = x[:, :, sel].mean(axis=2)  # .mean(['time'])
    want = (tm * w).sum(axis=-1) / w.sum()  # .weighted(weights).mean(lat)
    got = out[name]
    assert got.dims == ('realization', 'prediction_timedelta', 'level',
                        'longitude')
    assert got.values.dtype == np.float64
    np.testing.assert_allclose(got.values, want, rtol=1e-5, atol=1e-8)
  # K R K R: time and latitude are two runs, read in place
  assert fake.calls[0][1] == (33, 31, 108, 19, 1) and fake.calls[0][3]


# -- the operators end to end ---------------------------------------------------
def _dataset(dtype=np.float32):
  rs = np.random.RandomState(3)
  x = rs.standard_normal((5, 4, 3, 6)).astype(dtype)
  x[1, 2, 0, :2] = np.nan
  x[3, 0, 1, 4] = np.inf
  coords = {'time': pd.date_range('2020-01-01', periods=5).values,
            'level': np.array([500.0, 700.0, 850.0, 1000.0]),
            'latitude': np.array([-60.0, 0.0, 60.0]),
            'longitude': np.arange(6.0) * 60,
            'land': (('latitude', 'longitude'), rs.uniform(size=(3, 6)))}
  dims = ('time', 'level', 'latitude', 'longitude')
  return xl.Dataset({'t': (dims, x, {'units': 'K'})}, coords,
                    {'title': 'x'}), x


DIMS = ('time', 'level', 'latitude', 'longitude')


@pytest.mark.parametrize('avg,shape', [
    (['time', 'latitude'], (1, 5, 4, 3, 6)),
    (['longitude', 'level'], (5, 4, 3, 6, 1)),
    (['time', 'level', 'latitude', 'longitude'], (1, 360, 1, 1, 1)),
    (['level'], (5, 4, 1, 1, 18)),
    (['latitude', 'longitude'], (20, 18, 1, 1, 1)),
    (['time'], (1, 5, 1, 1, 72))])
@pytest.mark.parametrize('skipna', [False, True])
def test_compute_averages_layouts(avg, shape, skipna):
  ds, x = _dataset()
  with fake_ctx_average.installed() as fake:
    out = pp.compute_averages(ds, avg, skipna=skipna)
  keep = tuple(d for d in DIMS if d not in avg)
  t = out['t']
  assert t.dims == keep and t.attrs == {} and out.attrs == {}
  axes = [DIMS.index(d) for d in avg]
  weighted = 'latitude' in avg
  w = metrics.get_lat_weights(ds).values if weighted else None
  want = ao.average(x, axes, skipna, w, DIMS.index('latitude'))[0]
  assert _bits_equal(t.values, want)
  assert t.values.dtype == (np.float64 if weighted else np.float32)
  for name in DIMS:
    assert (name in out.coords) == (name not in avg)
  assert ('land' in out.coords) == (not {'latitude', 'longitude'} & set(avg))
  assert fake.calls[0][0] == 'average_host' and fake.calls[0][1] == shape
  assert fake.calls[0][5] == pp.AVERAGE_STREAM_BUDGET_BYTES


def test_three_runs_take_one_transposed_copy():
  rs = np.random.RandomState(5)
  x = rs.standard_normal((3, 4, 5, 6, 7)).astype(np.float64)
  dims = ('a', 'b', 'latitude', 'd', 'e')
  ds = xl.Dataset({'v': (dims, x)}, {'latitude': np.linspace(-80, 80, 5)})
  with fake_ctx_average.installed() as fake:
    out = pp.compute_averages(ds, ['a', 'latitude', 'e'])
  assert out['v'].dims == ('b', 'd')
  w = metrics.get_lat_weights(ds).values
  want = ao.average(x, [0, 2, 4], False, w, 2)[0]
  assert _bits_equal(out['v'].values, want)
  # R K after the copy; the weight index divides by the 7 'e' samples
  assert fake.calls[0][1] == (1, 105, 1, 1, 24) and fake.calls[0][4] == 7


def test_selection():
  ds, x = _dataset()
  with fake_ctx_average.installed():
    out = pp.compute_averages(ds, ['time'], variables=['t'],
                              levels=['850', 500], time_start='2020-01-02',
                              time_stop='2020-01-04')
    np.testing.assert_array_equal(out.coords['level'].values, [850.0, 500.0])
    want = ao.average(x[1:4][:, [2, 0]], [0])[0]
    assert _bits_equal(out['t'].values, want)
    out = pp.compute_averages(ds, ['level'], time_start='2021-01-01')
  assert out['t'].shape == (0, 3, 6)


def test_moment_reduce():
  ds, x = _dataset(np.float64)
  with fake_ctx_average.installed():
    got = {o: pp.moment_reduce(ds, o) for o in pp.MOMENT_ORDERS}
    sel = pp.moment_reduce(ds, 'first', ('time',), {'level': [700.0]})
  m, q, fr = ao.average(x, [2, 3], skipna=True)
  assert _bits_equal(got['zeroth']['t'].values, fr)
  assert _bits_equal(got['first']['t'].values, m)
  assert _bits_equal(got['second']['t'].values, q)
  for o in pp.MOMENT_ORDERS:
    assert got[o]['t'].dims == ('time', 'level')
  with np.errstate(invalid='ignore'):
    np.testing.assert_allclose(got['first']['t'].values,
                               np.nanmean(x, axis=(2, 3)))
    np.testing.assert_allclose(got['second']['t'].values,
                               np.nanmean(np.square(x), axis=(2, 3)))
  np.testing.assert_array_equal(got['zeroth']['t'].values,
                                np.mean(~np.isnan(x), axis=(2, 3)))
  assert sel['t'].dims == ('level', 'latitude', 'longitude')
  assert _bits_equal(sel['t'].values, ao.average(x[:, [1]], [0], True)[0])
  with pytest.raises(NotImplementedError, match='third'):
    pp.moment_reduce(ds, 'third')


def test_compute_statistical_moments():
  rs = np.random.RandomState(9)
  times = pd.date_range('2019-12-30', periods=6).values
  x = rs.standard_normal((6, 2, 3, 4)).astype(np.float32)
  x[2] = np.nan  # an all-NaN step: NaN moments that the time mean skips
  x[4, 1, 0, :3] = np.nan
  ds = xl.Dataset({'z': (('time', 'level', 'longitude', 'latitude'), x)},
                  {'time': times, 'level': np.array([500.0, 850.0]),
                   'longitude': np.arange(3.0), 'latitude': np.arange(4.0)})
  with fake_ctx_average.installed() as fake:
    out = pp.compute_statistical_moments(ds, start_year=2020, end_year=2020)
  assert list(out.keys()) == ['z_zeroth', 'z_first', 'z_second']
  sel = x[2:]  # 2020-01-01 .. 2020-01-04
  m, q, fr = ao.average(sel, [2, 3], skipna=True)
  for name, s in (('z_zeroth', fr), ('z_first', m), ('z_second', q)):
    v = out[name]
    assert v.dims == ('moment', 'level') and v.shape == (1, 2)
    want = ao.average(s, [0], skipna=True)[0]
    assert _bits_equal(v.values[0], want)
  assert out['z_first'].values.dtype == np.float32
  assert out['z_zeroth'].values.dtype == np.float64
  assert np.isfinite(out['z_first'].values).all()
  assert 'moment' not in out.coords and 'time' not in out.coords
  np.testing.assert_array_equal(out.coords['level'].values, [500.0, 850.0])
  # one spatial read per variable, then one small time mean per order
  assert [c[1] for c in fake.calls] == [(8, 12, 1, 1, 1)] + [(1, 4, 1, 1, 2)] * 3


def test_errors():
  ds, _ = _dataset()
  with fake_ctx_average.installed() as fake:
    bad = xl.Dataset({'i': (('x',), np.arange(4))})
    for fn in (lambda d: pp.compute_averages(d, ['x']),
               lambda d: pp.moment_reduce(d, 'first', ('x',))):
      with pytest.raises(TypeError, match="'i'"):
        fn(bad)
    two = xl.Dataset({'t': (DIMS, np.zeros((2, 1, 3, 4), np.float32)),
                      'z': (('latitude', 'longitude'),
                            np.zeros((3, 4), np.float32))},
                     {'time': pd.date_range('2020-01-01', periods=2).values})
    with pytest.raises(ValueError, match="'z'.*'time'"):
      pp.compute_averages(two, ['time'])
    with pytest.raises(ValueError, match="'z'.*'time'"):
      pp.compute_statistical_moments(two, start_year=None)
    with pytest.raises(ValueError, match='empty'):
      pp.compute_averages(ds, [])
    with pytest.raises(ValueError, match='empty'):
      pp.moment_reduce(ds, 'first', ())
    empty = xl.Dataset({'e': (('time', 'x'), np.zeros((0, 3), np.float32))})
    with pytest.raises(ValueError, match='empty'):
      pp.moment_reduce(empty, 'first', ('time',))
    assert not fake.calls
    # the entries' own checks
    ctx = _lib.default_context()
    x = np.zeros((2, 4, 3), np.float32)
    o = np.zeros(6, np.float32)
    good = dict(x=x.ctypes.data, dtype=_lib.F32, shape=(2, 4, 3, 1, 1),
                skipna=False, mean=o.ctypes.data)
    w = np.ones(3)
    for change, name in ((dict(dtype=5), 'dtype'),
                         (dict(shape=(2, 0, 3, 1, 1)), 'r0 and r1'),
                         (dict(shape=(2, 4, -3, 1, 1)), 'kept extents'),
                         (dict(weights=w), 'weights'),
                         (dict(weights=np.ones(2), wdiv=3), 'weights'),
                         (dict(mean=0), 'no output')):
      with pytest.raises(_lib.Wb2Error, match=name):
        ctx.average(**dict(good, **change))
      with pytest.raises(_lib.Wb2Error, match=name):
        ctx.average_host(**dict(good, budget=1 << 20, **change))

"""Time resampling and rolling windows without a GPU: the float64 oracle
(tests/resample_oracle.py) pinned to the reference test's known answers and to
cases derived by hand, pandas as an independent check where it agrees with
xarray, the bin tables, every error of the reference, and the operator layer
of weatherbench2_b200.resampling end to end on `fake_ctx_resample` (NumPy
interpreting the C-ABI arguments).  tests/test_resample_gpu.py runs the same
operator cases through the CUDA kernels."""
import numpy as np
import pandas as pd
import pytest

import resample_oracle as ro

DAY = pd.Timedelta('1D')


def _lite(values, times, dim='time'):
  from weatherbench2_b200 import xarray_lite as xl
  return xl.Dataset({'temperature': ((dim,), np.asarray(values))},
                    {dim: np.asarray(times)})


def _fake_run(fn, *args, **kw):
  import fake_ctx_resample
  with fake_ctx_resample.installed() as fake:
    return fn(*args, **kw), fake


def assert_matches(got, want, statistic, x, axis):
  """NaN masks identical; min / max exact; mean / sum within rtol 2e-6
  (float32) or 1e-12 (float64) plus an atol of 1e-6 (float32) or 1e-12
  (float64) times the largest |x| of the cell's series."""
  x = np.asarray(x)
  got = np.asarray(got)
  assert got.dtype == x.dtype, (got.dtype, x.dtype)
  got64 = got.astype(np.float64)
  want = np.asarray(want, np.float64)
  np.testing.assert_array_equal(np.isnan(got64), np.isnan(want),
                                err_msg=f'{statistic}: NaN mask')
  if statistic in ('min', 'max'):
    np.testing.assert_array_equal(got, want.astype(x.dtype), err_msg=statistic)
    return
  f32 = x.dtype == np.float32
  rtol = 2e-6 if f32 else 1e-12
  ax = np.abs(x.astype(np.float64))
  scale = np.max(np.where(np.isfinite(ax), ax, 0.0), axis=axis, keepdims=True)
  atol = (1e-6 if f32 else 1e-12) * np.broadcast_to(scale, want.shape)
  inf = np.isinf(want)
  np.testing.assert_array_equal(got64[inf], want[inf], err_msg=statistic)
  ok = np.isfinite(want)
  err = np.abs(got64 - want)[ok]
  bound = (atol + rtol * np.abs(want))[ok]
  assert (err <= bound).all(), (statistic, float((err / bound).max()))


# -- the oracle against the reference test's known answers -----------------------
@pytest.mark.parametrize('insert_nan', [False, True], ids=['NoNaN', 'YesNaN'])
def test_resample_and_rolling_are_aligned(insert_nan):
  """resample_in_time_test.py:34-117."""
  from weatherbench2_b200 import resampling
  times = pd.date_range('2023-01-01', periods=10)
  x = np.arange(10).astype(float)
  if insert_nan:
    x[0] = np.nan
  res, _ = _fake_run(resampling.resample_in_time, _lite(x, times), period='3d',
                     mean_vars=['ALL'])
  np.testing.assert_array_equal(
      pd.to_datetime(res.coords['time'].values),
      pd.DatetimeIndex(['2023-01-01', '2023-01-04', '2023-01-07', '2023-01-10']))
  want = [np.mean(x[:3]), np.mean(x[3:6]), np.mean(x[6:9]), np.mean(x[9:12])]
  np.testing.assert_array_equal(res['temperature'].values, want)
  np.testing.assert_array_equal(ro.resample(x, [0, 3, 6, 9], [3, 3, 3, 1],
                                            ['mean'])['mean'], want)
  roll, _ = _fake_run(resampling.resample_in_time, _lite(x, times),
                      period='3d', method='rolling', mean_vars=['ALL'])
  rt = pd.to_datetime(roll.coords['time'].values)
  for i, t in enumerate(pd.DatetimeIndex(['2023-01-01', '2023-01-04',
                                          '2023-01-07'])):
    np.testing.assert_array_equal(roll['temperature'].values[rt.get_loc(t)],
                                  want[i])


ALIGNED_CASES = [(20, '3d', None), (21, '3d', None), (21, '8d', None),
                 (5, '1d', None), (20, '3d', [0, 4, 8]), (21, '3d', [20]),
                 (21, '8d', [15])]


def aligned_case(case):
  """resample_in_time_test.py:119-189: (resample, rolling) of one case."""
  from weatherbench2_b200 import resampling
  n, period, nans = case
  times = pd.date_range('2010', periods=n)
  x = np.random.RandomState(802701).rand(n)
  for i in nans or []:
    x[i] = np.nan
  ds = _lite(x, times)
  return (resampling.resample_in_time(ds, period=period, mean_vars=['ALL']),
          resampling.resample_in_time(ds, period=period, method='rolling',
                                      mean_vars=['ALL']), x)


def check_aligned(res, roll, rtol=0.0):
  """Equal values (within `rtol`) and NaN masks at the common times."""
  rt = pd.to_datetime(res.coords['time'].values)
  common = rt.intersection(pd.to_datetime(roll.coords['time'].values))
  assert len(common) >= len(rt) - 1
  a = res['temperature'].values[rt.get_indexer(common)]
  b = roll['temperature'].values[pd.to_datetime(
      roll.coords['time'].values).get_indexer(common)]
  np.testing.assert_array_equal(np.isnan(a), np.isnan(b))
  np.testing.assert_allclose(np.asarray(a), np.asarray(b), rtol=rtol, atol=0)


@pytest.mark.parametrize('case', ALIGNED_CASES, ids=str)
def test_resample_equals_rolling_on_common_times(case):
  import fake_ctx_resample
  with fake_ctx_resample.installed():
    res, roll, _ = aligned_case(case)
  check_aligned(res, roll)


# -- the oracle against cases derived by hand -------------------------------------
def test_empty_bins_are_nan_for_every_statistic():
  times = pd.DatetimeIndex(['2023-01-01 06:00', '2023-01-02', '2023-01-05',
                            '2023-01-06'])
  from weatherbench2_b200 import resampling
  labels, start, count = resampling._bins(times, DAY, 'left')  # pylint: disable=protected-access
  np.testing.assert_array_equal(count, [1, 1, 0, 0, 1, 1])
  np.testing.assert_array_equal(start, [0, 1, 2, 2, 2, 3])
  assert labels.size == 6
  x = np.array([1.0, 2.0, 3.0, 4.0])
  for skipna in (False, True):
    got = ro.resample(x, start, count, skipna=skipna)
    for s in ro.STATISTICS:
      np.testing.assert_array_equal(got[s], [1, 2, np.nan, np.nan, 3, 4])


def test_all_nan_bin_under_each_skipna():
  x = np.array([np.nan, np.nan, 1.0, np.nan, 3.0])
  start, count = [0, 2], [2, 3]
  got = ro.resample(x, start, count, skipna=False)
  for s in ro.STATISTICS:
    np.testing.assert_array_equal(got[s], [np.nan, np.nan])
  got = ro.resample(x, start, count, skipna=True)
  np.testing.assert_array_equal(got['mean'], [np.nan, 2.0])
  np.testing.assert_array_equal(got['min'], [np.nan, 1.0])
  np.testing.assert_array_equal(got['max'], [np.nan, 3.0])
  np.testing.assert_array_equal(got['sum'], [0.0, 4.0])


def test_inf_entering_and_leaving_a_rolling_window():
  inf = np.inf
  got = ro.rolling(np.array([1.0, inf, 2.0, 3.0, 4.0]), 2)
  np.testing.assert_array_equal(got['sum'], [np.nan, inf, inf, 5, 7])
  np.testing.assert_array_equal(got['mean'], [np.nan, inf, inf, 2.5, 3.5])
  np.testing.assert_array_equal(got['max'], [np.nan, inf, inf, 3, 4])
  got = ro.rolling(np.array([1.0, inf, -inf, 3.0, 5.0]), 2)
  np.testing.assert_array_equal(got['sum'], [np.nan, inf, np.nan, -inf, 8])
  np.testing.assert_array_equal(got['min'], [np.nan, 1, -inf, -inf, 3])


def test_window_one_and_window_longer_than_the_series():
  x = np.array([1.0, np.nan, 3.0])
  for s, v in ro.rolling(x, 1).items():
    np.testing.assert_array_equal(v, x, err_msg=s)
  for v in ro.rolling(x[[0, 2]], 3).values():
    assert np.isnan(v).all()


# -- pandas as an independent check ------------------------------------------------
@pytest.mark.parametrize('period', ['3D', '7D', '10h'])
def test_bins_and_nan_free_resample_match_pandas(period):
  from weatherbench2_b200 import resampling
  times = pd.date_range('2020-01-01 03:00', periods=50, freq='6h')
  x = np.random.RandomState(0).normal(size=50)
  labels, start, count = resampling._bins(times, pd.Timedelta(period), 'left')  # pylint: disable=protected-access
  got = ro.resample(x, start, count)
  want = pd.Series(x, index=times).resample(pd.Timedelta(period))
  np.testing.assert_array_equal(pd.DatetimeIndex(labels), want.mean().index)
  for s in ro.STATISTICS:
    w = getattr(want, s)().to_numpy()
    if s == 'sum':
      w = np.where(count == 0, np.nan, w)  # pandas' empty-bin sum is 0
    np.testing.assert_allclose(got[s], w, rtol=1e-12, err_msg=s)


def test_rolling_with_nan_matches_pandas():
  x = np.random.RandomState(1).normal(size=40)
  x[[3, 17, 18]] = np.nan
  for w in (1, 4, 9):
    got = ro.rolling(x, w)
    r = pd.Series(x).rolling(w, min_periods=w)
    for s in ro.STATISTICS:
      np.testing.assert_allclose(got[s], getattr(r, s)().to_numpy(),
                                 rtol=1e-12, err_msg=(w, s))


def test_bin_tables_on_a_timedelta_index_and_the_right_label_side():
  from weatherbench2_b200 import resampling
  t = pd.timedelta_range('0 days', periods=10, freq='1D')
  labels, start, count = resampling._bins(t, 3 * DAY, 'left')  # pylint: disable=protected-access
  np.testing.assert_array_equal(pd.TimedeltaIndex(labels),
                                pd.to_timedelta([0, 3, 6, 9], 'D'))
  np.testing.assert_array_equal(start, [0, 3, 6, 9])
  np.testing.assert_array_equal(count, [3, 3, 3, 1])
  # origin = the first value of a timedelta axis
  labels, _, _ = resampling._bins(t + DAY, 3 * DAY, 'left')  # pylint: disable=protected-access
  np.testing.assert_array_equal(pd.TimedeltaIndex(labels),
                                pd.to_timedelta([1, 4, 7, 10], 'D'))
  # right: (T - period, T] labelled T, the first bin dropped
  labels, start, count = resampling._bins(t, 3 * DAY, 'right')  # pylint: disable=protected-access
  np.testing.assert_array_equal(pd.TimedeltaIndex(labels),
                                pd.to_timedelta([3, 6, 9, 12], 'D'))
  np.testing.assert_array_equal(start, [1, 4, 7, 10])
  np.testing.assert_array_equal(count, [3, 3, 3, 0])
  d = pd.date_range('2023-01-01', periods=10)
  labels, start, count = resampling._bins(d, 3 * DAY, 'right')  # pylint: disable=protected-access
  np.testing.assert_array_equal(
      pd.DatetimeIndex(labels),
      pd.DatetimeIndex(['2023-01-04', '2023-01-07', '2023-01-10']))
  np.testing.assert_array_equal(start, [1, 4, 7])
  np.testing.assert_array_equal(count, [3, 3, 3])


# -- the operator layer end to end ------------------------------------------------------
OPERATOR_CASES = [(f'{dim}-{method}-{period}-{suffix}', dim, method, period,
                   suffix)
                  for dim in ('time', 'prediction_timedelta')
                  for method, suffix, period in (
                      ('resample', False, '5d'), ('resample', True, '1w'),
                      ('resample', True, '1d'), ('rolling', True, '1w'),
                      ('rolling', False, '30d'), ('rolling', True, '1d'))]


def operator_dataset(dim):
  """Daily truth (time, level, latitude, longitude) over 2021, or a forecast
  (time, prediction_timedelta, level, longitude, latitude) with 16 daily leads;
  temperature float32, geopotential float64 (+ 10), two variables to drop."""
  from weatherbench2_b200 import xarray_lite as xl
  rs = np.random.RandomState(5)
  lat, lon, level = np.linspace(-90, 90, 7), np.arange(0, 360, 30.0), np.array(
      [500, 700, 850])
  if dim == 'time':
    times = pd.date_range('2021-01-01', '2022-01-01', freq='1D').values
    dims = ('time', 'level', 'latitude', 'longitude')
    coords = dict(time=times, level=level, latitude=lat, longitude=lon)
  else:
    times = pd.date_range('2021-01-01', '2021-01-10', freq='1D').values
    lead = pd.timedelta_range('0 day', '15 days', freq='1D').values
    dims = ('time', 'prediction_timedelta', 'level', 'longitude', 'latitude')
    coords = dict(time=times, prediction_timedelta=lead, level=level,
                  longitude=lon, latitude=lat)
  shape = tuple(np.asarray(coords[d]).size for d in dims)
  return xl.Dataset({
      'temperature': (dims, rs.normal(size=shape).astype(np.float32)),
      'geopotential': (dims, rs.normal(size=shape) + 10),
      'should_drop': (dims, rs.normal(size=shape).astype(np.float32)),
      'var_to_drop': (('dim_to_drop',), np.ones(5)),
  }, coords)


def run_operator_case(case, convert=None):
  """resample_in_time over the structure of resample_in_time_test.py:229-342
  (time) and :382-503 (prediction_timedelta) against the oracle; returns the
  result.  `convert` maps the input dataset (e.g. to device tensors)."""
  from weatherbench2_b200 import resampling
  _, dim, method, period, suffix = case
  ds = operator_dataset(dim)
  start, stop = (('2021-02-01', '2021-04-01') if dim == 'time' else
                 ('0 day', '9 days'))
  got = resampling.resample_in_time(
      convert(ds) if convert else ds, period=period, method=method,
      mean_vars=['temperature', 'geopotential'],
      min_vars=['temperature', 'geopotential'], max_vars=['temperature'],
      sum_vars=['geopotential'], add_mean_suffix=suffix, time_start=start,
      time_stop=stop, time_dim=dim)
  m = '_mean' if suffix else ''
  assert sorted(got.keys()) == sorted([
      f'temperature{m}', f'geopotential{m}', 'temperature_min',
      'geopotential_min', 'temperature_max', 'geopotential_sum'])
  index = pd.Index(ds.coords[dim].values)
  sel = np.arange(index.size)[index.slice_indexer(start, stop)]
  t = index[sel]
  p = pd.Timedelta(period)
  axis = ds['temperature'].dims.index(dim)
  if method == 'resample':  # origin start_day (datetime) / first value
    origin = t[0].floor('D') if dim == 'time' else t[0]
    k = np.asarray((t - origin) // p)
    count = np.bincount(k)
    start_pos = np.cumsum(count) - count
    want_t = origin + p * np.arange(count.size)
  else:
    w = p // DAY
    want_t = t - p + DAY
  np.testing.assert_array_equal(np.asarray(got.coords[dim].values),
                                np.asarray(want_t))
  for name in ('temperature', 'geopotential'):
    x = np.take(ds[name].values, sel, axis=axis)
    stats = {'temperature': ('mean', 'min', 'max'),
             'geopotential': ('mean', 'min', 'sum')}[name]
    want = (ro.resample(x, start_pos, count, stats, axis=axis)
            if method == 'resample' else ro.rolling(x, w, stats, axis=axis))
    for s in stats:
      key = f'{name}{m}' if s == 'mean' else f'{name}_{s}'
      da = got[key]
      assert da.dims == ds[name].dims
      assert_matches(da.values, want[s], s, x, axis)
    if period != '1d':
      mean = got[f'{name}{m}'].values
      ok = ~np.isnan(mean)
      assert (got[f'{name}_min'].values[ok] < mean[ok]).all()
      if name == 'temperature':
        assert (mean[ok] < got['temperature_max'].values[ok]).all()
  assert 'dim_to_drop' not in got.sizes
  return got


@pytest.mark.parametrize('case', OPERATOR_CASES, ids=[c[0] for c in
                                                       OPERATOR_CASES])
def test_resample_in_time_matches_the_oracle(case):
  _, fake = _fake_run(run_operator_case, case)
  # one read per variable: all statistics of a variable in one call
  assert len(fake.calls) == 2


def test_resample_in_time_core_on_a_dataset_and_a_dataarray():
  from weatherbench2_b200 import resampling
  times = pd.date_range('2023-01-01', periods=10)
  x = np.arange(10.0)
  ds = _lite(x, times)
  ds['const'] = (('other',), np.ones(3))
  got, _ = _fake_run(resampling.resample_in_time_core, ds, 'resample', '3d',
                     'sum', False)
  np.testing.assert_array_equal(got['temperature'].values, [3, 12, 21, 9])
  np.testing.assert_array_equal(got['const'].values, np.ones(3))
  got, _ = _fake_run(resampling.resample_in_time_core, ds['temperature'],
                     'rolling', '2d', 'max', False)
  np.testing.assert_array_equal(got.values, [np.nan] + list(range(1, 10)))
  got, _ = _fake_run(resampling.resample_in_time_core, ds, 'resample', '3d',
                     'min', False, label_side='right')
  np.testing.assert_array_equal(got['temperature'].values, [1, 4, 7])


# -- errors ---------------------------------------------------------------------------
def test_errors_of_the_reference():
  from weatherbench2_b200 import resampling
  times = pd.date_range('2023-01-01', periods=10)
  ds = _lite(np.arange(10.0), times)
  ds['const'] = (('other',), np.ones(3))
  core = resampling.resample_in_time_core
  main = resampling.resample_in_time
  with pytest.raises(ValueError, match='did not evenly divide'):
    _fake_run(core, ds, 'rolling', '36h', 'mean', False)
  with pytest.raises(ValueError, match='Unhandled method'):
    _fake_run(core, ds, 'nearest', '3d', 'mean', False)
  with pytest.raises(ValueError, match='Unhandled label_side'):
    _fake_run(core, ds, 'resample', '3d', 'mean', False, label_side='middle')
  with pytest.raises(ValueError, match='Unhandled label_side'):
    _fake_run(main, ds, period='3d', method='rolling', mean_vars=['ALL'],
              label_side='middle')
  with pytest.raises(ValueError, match='Cannot specify both ALL'):
    _fake_run(main, ds, period='3d', mean_vars=['ALL', 'temperature'])
  with pytest.raises(ValueError, match='did not contain time'):
    _fake_run(main, ds, period='3d', max_vars=['const'])
  gap = _lite(np.arange(3.0), pd.DatetimeIndex(['2023-01-01', '2023-01-02',
                                                '2023-01-04']))
  with pytest.raises(ValueError, match='constant spacing'):
    _fake_run(main, gap, period='2d', method='rolling', mean_vars=['ALL'])
  back = _lite(np.arange(3.0), times[[0, 2, 1]])
  with pytest.raises(ValueError, match='monotonic'):
    _fake_run(main, back, period='2d', mean_vars=['ALL'])
  ints = _lite(np.arange(10, dtype=np.int32), times)
  with pytest.raises(TypeError, match="'temperature'"):
    _fake_run(main, ints, period='2d', sum_vars=['temperature'])

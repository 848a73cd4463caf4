"""Day-of-year climatologies without a GPU: the float64 oracle
(tests/climatology_oracle.py) pinned to answers derived by hand, the error
cases of the reference, and the operator layer of weatherbench2_b200.utils end
to end on `fake_ctx_climatology` (NumPy interpreting the C-ABI tables) against
the oracle.  tests/test_climatology_gpu.py runs the same operator cases through
the CUDA kernels."""
import numpy as np
import pandas as pd
import pytest

import climatology_oracle as co

H = np.timedelta64(1, 'h')


def _times(start, stop, step_h):
  return np.arange(np.datetime64(start, 'ns'), np.datetime64(stop, 'ns'),
                   np.timedelta64(step_h, 'h').astype('timedelta64[ns]'))


def _circular(values, window_size):
  """sum_j w[j] values[(d + j) mod N] / window_size, by hand."""
  w = co.window_weights(window_size)
  half = window_size // 2
  n = len(values)
  return np.array([sum(w[j + half] * values[(d + j) % n]
                       for j in range(-half, half + 1)) / window_size
                   for d in range(n)])


# -- the oracle against answers derived by hand ---------------------------------
def test_window_weights_are_triangular_with_mean_one():
  w = co.window_weights(61)
  assert w.size == 61 and w[0] == 0 and w[-1] == 0
  np.testing.assert_allclose(w.mean(), 1.0)
  np.testing.assert_allclose(w[30], 61 / 30)
  with pytest.raises(AssertionError):
    co.window_weights(60)


@pytest.mark.parametrize('method', ['explicit', 'fast'])
def test_constant_field_gives_its_value_and_zero_std(method):
  t = _times('2019-01-01', '2021-01-01', 6)
  x = np.full((t.size, 3), 7.25)
  fn = co.hourly_stat if method == 'explicit' else co.hourly_stat_fast
  for stat, want in (('mean', 7.25), ('std', 0.0)):
    labels, v = fn(t, x, 61, slice('2019', '2020'), 6, stat)
    assert labels.size == 366 and v.shape == (4, 366, 3)
    np.testing.assert_allclose(v, want, atol=1e-12)


def test_two_constant_years_give_half_their_difference_as_std():
  t = _times('2021-01-01', '2023-01-01', 24)
  x = np.where(pd.DatetimeIndex(t).year == 2021, 3.0, -1.0)[:, None]
  labels, v = co.hourly_stat(t, x, 61, slice('2021', '2022'), 24, 'std')
  assert labels.size == 365
  np.testing.assert_allclose(v, 2.0, rtol=1e-12)
  _, m = co.hourly_stat(t, x, 61, slice('2021', '2022'), 24, 'mean')
  np.testing.assert_allclose(m, 1.0, rtol=1e-12)


def test_impulse_gives_the_shifted_window_weights_with_wrap_around():
  years, d0 = 3, 2  # day label 3: the window wraps into December
  t = _times('2021-01-01', '2024-01-01', 24)
  ti = pd.DatetimeIndex(t)
  x = np.zeros((t.size, 1))
  x[(ti.year == 2021) & (ti.dayofyear == d0 + 1)] = 1.0
  _, v = co.hourly_stat(t, x, 61, slice('2021', '2023'), 24, 'mean')
  w = co.window_weights(61)
  want = np.zeros(365)
  for j in range(-30, 31):  # out[d] = w[j] / (61 Y) at d = d0 - j (mod 365)
    want[(d0 - j) % 365] += w[j + 30] / (61 * years)
  np.testing.assert_allclose(v[0, :, 0], want, atol=1e-15)


def test_reference_claim_explicit_equals_fast_for_dayofyear_truth():
  """utils_test.py:24-47: 2022, daily, truth = dayofyear, hour_interval 24."""
  t = _times('2022-01-01', '2023-01-01', 24)
  x = np.asarray(pd.DatetimeIndex(t).dayofyear, np.float64)[:, None]
  _, explicit = co.hourly_stat(t, x, 61, slice('2022', '2022'), 24, 'mean')
  _, fast = co.hourly_stat_fast(t, x, 61, slice('2022', '2022'), 24, 'mean')
  want = _circular(np.arange(1, 366, dtype=np.float64), 61)
  np.testing.assert_allclose(explicit[0, :, 0], want, rtol=1e-12)
  np.testing.assert_allclose(fast[0, :, 0], want, rtol=1e-12)


def test_rule1_leap_year_beside_non_leap_year_fills_day_366():
  t = _times('2019-01-01', '2021-01-01', 24)
  x = np.where(pd.DatetimeIndex(t).year == 2019, 1.0, 5.0)[:, None]
  labels, m = co.hourly_stat(t, x, 61, slice('2019', '2020'), 24, 'mean')
  _, s = co.hourly_stat(t, x, 61, slice('2019', '2020'), 24, 'std')
  # day 366 of 2019 is 2019's day 365: every day sees both years equally
  assert labels.size == 366
  np.testing.assert_allclose(m, 3.0, rtol=1e-12)
  np.testing.assert_allclose(s, 2.0, rtol=1e-12)
  labels, _ = co.hourly_stat(t[:365], x[:365], 61, slice('2019', '2019'), 24,
                             'mean')
  assert labels.size == 365


def _filled_by_hand(t, x, nan_pos):
  """The same series with the NaN replaced by its year's day-365 value."""
  ti = pd.DatetimeIndex(t)
  y = x.copy()
  for p in nan_pos:
    src = (ti.year == ti.year[p]) & (ti.dayofyear == 365)
    y[p] = np.where(np.isnan(x[p]), x[src][0], x[p])
  return y


def test_rule2_nan_on_an_ordinary_day_takes_that_years_day_365():
  t = _times('2021-01-01', '2023-01-01', 24)
  rs = np.random.RandomState(0)
  x = rs.normal(size=(t.size, 2))
  x[100, 0] = np.nan
  want = _filled_by_hand(t, x, [100])
  assert want[100, 0] == x[364, 0]
  for stat in ('mean', 'std'):
    _, got = co.hourly_stat(t, x, 11, slice('2021', '2022'), 24, stat)
    _, ref = co.hourly_stat(t, want, 11, slice('2021', '2022'), 24, stat)
    np.testing.assert_allclose(got, ref, rtol=1e-12)


def test_rule2_partial_first_year_and_missing_day_365():
  t = _times('2021-07-19', '2023-01-01', 24)  # 2021 starts at day 200
  rs = np.random.RandomState(1)
  x = rs.normal(size=(t.size, 1))
  _, got = co.hourly_stat(t, x, 61, slice('2021', '2022'), 24, 'mean')
  # by hand: 2021's days 1..199 hold 2021's day-365 value
  ti = pd.DatetimeIndex(t)
  d365 = x[(ti.year == 2021) & (ti.dayofyear == 365)][0, 0]
  y21 = np.full(365, d365)
  y21[199:] = x[ti.year == 2021, 0]
  y22 = x[ti.year == 2022, 0]
  want = (_circular(y21, 61) + _circular(y22, 61)) / 2
  np.testing.assert_allclose(got[0, :, 0], want, rtol=1e-12)
  with pytest.raises(KeyError):  # no day labelled 365 at all
    co.hourly_stat(t[:100], x[:100], 61, slice('2021', '2021'), 24, 'mean')


def test_rule4_fast_method_divides_by_the_count_of_valid_taps():
  t = _times('2021-01-01', '2022-01-01', 24)
  x = np.full((t.size, 1), 2.0)
  x[50] = np.nan  # day label 51 has no value at all
  _, m = co.hourly_stat_fast(t, x, 61, slice('2021', '2021'), 24, 'mean')
  w = co.window_weights(61)
  # on the NaN day the centre tap (weight 61/30) is missing: 60 valid taps
  np.testing.assert_allclose(m[0, 50, 0], 2.0 * (61 - w[30]) / 60,
                             rtol=1e-12)
  np.testing.assert_allclose(m[0, 50 + 30, 0], 2.0 * (61 - w[0]) / 60,
                             rtol=1e-12)  # a zero-weight tap still counts
  np.testing.assert_allclose(m[0, 200, 0], 2.0, rtol=1e-12)


def test_rule5_daily_resample_creates_missing_days_and_fills_them():
  t = _times('2021-01-01', '2022-01-01', 6)
  ti = pd.DatetimeIndex(t)
  keep = ti.dayofyear != 50
  t, ti = t[keep], ti[keep]
  x = (np.asarray(ti.dayofyear, np.float64) +
       np.asarray(ti.hour) / 24.0)[:, None]
  days, daily = co.resample_daily(ti, x)
  assert days.size == 365 and np.isnan(daily[49, 0])
  np.testing.assert_allclose(daily[10, 0], 11 + 9 / 24)
  _, got = co.daily_stat(t, x, 61, slice('2021', '2021'), 'mean')
  series = np.arange(1, 366) + 9 / 24
  series[49] = 365 + 9 / 24  # the NaN day takes day 365
  np.testing.assert_allclose(got[:, 0], _circular(series, 61), rtol=1e-12)


# -- the operator layer on the NumPy stand-in of the C ABI ------------------------
def make_obs(layout='4d', dtype=np.float32, nan_frac=0.0, start='2019-03-10',
             stop='2021-02-01', step_h=6, seed=0, offset=0.0, noise=1.0):
  """A synthetic truth dataset with a seasonal cycle."""
  from weatherbench2_b200 import xarray_lite as xl
  t = _times(start, stop, step_h)
  ti = pd.DatetimeIndex(t)
  rs = np.random.RandomState(seed)
  lat, lon = np.linspace(-90, 90, 5), np.arange(4) * 90.0
  if layout == '4d':
    dims = ('time', 'level', 'longitude', 'latitude')
    other = (2, lon.size, lat.size)
    coords = dict(level=np.array([500, 850]), longitude=lon, latitude=lat)
  else:
    dims = ('time', 'latitude', 'longitude')
    other = (lat.size, lon.size)
    coords = dict(latitude=lat, longitude=lon)
  season = 10 * np.sin(2 * np.pi * np.asarray(ti.dayofyear) / 365.25 +
                       np.asarray(ti.hour) / 4)
  x = offset + season.reshape((-1,) + (1,) * len(other)) + noise * rs.normal(
      size=(t.size,) + other)
  if nan_frac:
    x[rs.uniform(size=x.shape) < nan_frac] = np.nan
  x = x.astype(dtype)
  ds = xl.Dataset({'z': (dims, x), 'orog': (dims[1:], x[0])},
                  dict(coords, time=t))
  return ds, t, x


# (name, make_obs kwargs, frequency, method, hour_interval, statistics, window)
OPERATOR_CASES = [
    ('hourly6_explicit_both_4d', {}, 'hourly', 'explicit', 6,
     ('mean', 'std'), 61),
    ('hourly12_explicit_mean_3d_nan', dict(layout='3d', nan_frac=0.05),
     'hourly', 'explicit', 12, ('mean',), 61),
    ('hourly6_fast_both_3d', dict(layout='3d'), 'hourly', 'fast', 6,
     ('mean', 'std'), 31),
    ('hourly12_fast_std_f64_nan', dict(dtype=np.float64, nan_frac=0.05),
     'hourly', 'fast', 12, ('std',), 61),
    ('hourly6_explicit_std_f64', dict(dtype=np.float64, layout='3d'),
     'hourly', 'explicit', 6, ('std',), 15),
    ('daily_explicit_both_nan', dict(nan_frac=0.05), 'daily', 'explicit',
     None, ('mean', 'std'), 61),
    ('daily_fast_mean_3d', dict(layout='3d'), 'daily', 'fast', None,
     ('mean',), 61),
    ('daily_fast_both_f64_nan', dict(dtype=np.float64, nan_frac=0.05),
     'daily', 'fast', None, ('mean', 'std'), 61),
]


def oracle_for(t, x, frequency, method, hour_interval, stat, window):
  years = slice('2019', '2020')
  if frequency == 'hourly':
    fn = co.hourly_stat if method == 'explicit' else co.hourly_stat_fast
    return fn(t, x, window, years, hour_interval, stat)
  fn = co.daily_stat if method == 'explicit' else co.daily_stat_fast
  return fn(t, x, window, years, stat)


def run_operator_case(case, obs_transform=lambda ds: ds):
  """Runs one OPERATOR_CASES entry through weatherbench2_b200.utils and
  compares with the oracle (rtol 1e-5, atol 1e-6 max|x|)."""
  from weatherbench2_b200 import utils
  _, kw, frequency, method, hour_interval, stats, window = case
  ds, t, x = make_obs(**kw)
  obs = obs_transform(ds)
  if len(stats) > 1:
    out = utils.compute_climatology(
        obs, frequency=frequency, hour_interval=hour_interval or 1,
        window_size=window, start_year=2019, end_year=2020, statistics=stats,
        method=method)
    got = {s: out['z' if s == 'mean' else 'z_std'] for s in stats}
    assert 'orog' not in out and 'orog_std' not in out
  else:
    years = slice('2019', '2020')
    if frequency == 'hourly':
      fn = (utils.compute_hourly_stat if method == 'explicit'
            else utils.compute_hourly_stat_fast)
      res = fn(obs, window, years, hour_interval, stats[0])
    else:
      fn = (utils.compute_daily_stat if method == 'explicit'
            else utils.compute_daily_stat_fast)
      res = fn(obs, window, years, stats[0])
    got = {stats[0]: res['z']}
  atol = 1e-6 * np.nanmax(np.abs(x))
  for s, da in got.items():
    labels, want = oracle_for(t, x.astype(np.float64), frequency, method,
                              hour_interval, s, window)
    lead = ('hour', 'dayofyear') if frequency == 'hourly' else ('dayofyear',)
    assert da.dims == lead + tuple(d for d in ds['z'].dims if d != 'time')
    np.testing.assert_array_equal(da.coords['dayofyear'].values, labels)
    if frequency == 'hourly':
      np.testing.assert_array_equal(da.coords['hour'].values,
                                    np.arange(0, 24, hour_interval))
    vals = da.values
    assert vals.dtype == np.float32
    np.testing.assert_allclose(vals, want, rtol=1e-5, atol=atol,
                               err_msg=f'{case[0]} {s}')
  return got


@pytest.mark.parametrize('case', OPERATOR_CASES, ids=[c[0] for c in
                                                       OPERATOR_CASES])
def test_operator_layer_matches_the_oracle_on_fake_ctx(case):
  import fake_ctx_climatology
  with fake_ctx_climatology.installed() as fake:
    run_operator_case(case)
  kinds = {c[0] for c in fake.calls}
  assert kinds == {'climatology_host'}
  # mean and std together: one call (one read of the input)
  if case[3] == 'explicit' or case[2] == 'hourly':
    assert len(fake.calls) == 1


def test_tables_stack_years_on_the_union_of_day_labels():
  from weatherbench2_b200 import utils
  t = _times('2019-01-01', '2021-01-01', 6)
  plan, labels = utils._plan(t, slice('2019', '2020'), [0, 12], utils.EXPLICIT,
                             False, 61)
  assert labels.size == 366 and plan.items.shape == (2, 366, 2)
  assert plan.items[0, 365, 0] == -1  # 2019 has no day 366
  assert plan.fill[0, 0] == plan.items[0, 364, 0]
  assert plan.items[1, 0, 1] == 365 * 4 + 2  # 2020-01-01T12
  plan, labels = utils._plan(t, slice('2019', '2020'), None, utils.FAST, False,
                             61)
  assert plan.items.shape == (1, 366, 8) and plan.nres == 0
  assert (plan.items[0, 365] >= 0).sum() == 4
  plan, labels = utils._plan(t, slice('2020', '2020'), None, utils.EXPLICIT,
                             True, 61)
  assert plan.nres == 366 and (plan.res_count == 4).all()
  assert plan.res_start[0] == 365 * 4


def test_error_cases_match_the_reference():
  import fake_ctx_climatology
  from weatherbench2_b200 import utils
  ds, _, _ = make_obs(stop='2019-06-01')
  with fake_ctx_climatology.installed():
    with pytest.raises(AssertionError):
      utils.compute_hourly_stat(ds, 60, slice('2019', '2019'), 6)
    with pytest.raises(AssertionError):
      utils.create_window_weights(4)
    with pytest.raises(KeyError):  # no day labelled 365
      utils.compute_hourly_stat(ds, 61, slice('2019', '2019'), 6)
    full, _, _ = make_obs(layout='3d')
    with pytest.raises(ValueError):  # 6-hourly data has no 03 UTC
      utils.compute_hourly_stat(full, 61, slice('2019', '2020'), 3)
    with pytest.raises(ValueError):
      utils.compute_hourly_stat_fast(ds, 61, slice('2030', '2031'), 6)
    for stat in ('seeps', 'quantile', 'median'):
      with pytest.raises(NotImplementedError, match='out of its scope'):
        utils.compute_climatology(ds, statistics=(stat,))
      with pytest.raises(NotImplementedError):
        utils.compute_daily_stat_fast(ds, 61, slice('2019', '2019'), stat)
    with pytest.raises(NotImplementedError):
      utils.compute_climatology(ds, frequency='monthly')


def test_create_window_weights_is_the_references():
  from weatherbench2_b200 import utils
  w = utils.create_window_weights(61)
  assert w.dims == ('window',)
  np.testing.assert_array_equal(w.values, co.window_weights(61))

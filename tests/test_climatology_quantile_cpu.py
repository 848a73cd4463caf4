"""Quantile and SEEPS day-of-year climatologies without a GPU: the float64
oracle (tests/climatology_quantile_oracle.py) pinned to answers derived by
hand, the new error cases, and the operators of weatherbench2_b200.utils end
to end on `fake_ctx_climatology_quantile` against the oracle.
tests/test_climatology_quantile_gpu.py runs the same cases through the CUDA
kernel."""
import numpy as np
import pandas as pd
import pytest

import climatology_oracle as co
import climatology_quantile_oracle as cq
from test_climatology_cpu import _times, make_obs


# -- the oracle against answers derived by hand ---------------------------------
def test_equal_weights_give_numpy_linear_quantiles():
  rs = np.random.RandomState(0)
  data = rs.normal(size=37)
  qs = np.array([0.0, 0.1, 0.37, 0.5, 2 / 3, 0.9, 1.0])
  got = cq.weighted_quantile(data, np.ones(37), qs)
  np.testing.assert_allclose(got, np.quantile(data, qs, method='linear'),
                             rtol=0, atol=1e-13)


def test_weighted_quantile_by_hand():
  # nw = 16 / 6, c = [0, .25, .5, 1], h = 11 / 6: v(c) = clip(8c/3 - 5/6, 0, 1)
  # = [0, 0, .5, 1], so 1 * 0 + 2 * .5 + 3 * .5 = 2.5
  got = cq.weighted_quantile([1, 2, 3, 4], [1, 1, 2, 0], 0.5)
  np.testing.assert_allclose(got, [2.5], rtol=1e-14)
  assert np.isnan(cq.weighted_quantile([np.nan, 1.0], [1, 0], 0.5)[0])


def test_reference_seeps_answer():
  """compute_climatology_test: [0, 0.25, 2, 4, 6] mm, threshold 0.25 mm."""
  x = np.array([0, 0.25, 2, 4, 6]) / 1000
  thr, frac = cq.seeps_of_window(x, np.ones(5), 0.25 / 1000)
  np.testing.assert_allclose(frac, 1 / 5)
  np.testing.assert_allclose(thr, 4e-3, rtol=1e-12)


def _alternating_year():
  """2021 daily: even day index dry (0), odd wet ((i + 1) mm)."""
  t = _times('2021-01-01', '2022-01-01', 24)
  i = np.arange(t.size)
  x = np.where(i % 2 == 0, 0.0, (i + 1) / 1000.0)[:, None]
  return t, x


def test_zero_weight_end_taps_count_only_in_the_dry_fraction():
  t, x = _alternating_year()
  _, thr, frac = cq.rolling_seeps(pd.DatetimeIndex(t), x, 3, 0.5 / 1000)
  # window 3: taps (0, 1, 0); a wet centre has two dry neighbours
  np.testing.assert_allclose(thr[101, 0], x[101, 0], rtol=1e-14)
  np.testing.assert_allclose(frac[101, 0], 2 / 3)
  # a dry centre: every weighted sample dry -> NaN; one dry sample in three
  assert np.isnan(thr[100, 0])
  np.testing.assert_allclose(frac[100, 0], 1 / 3)


def test_nan_is_not_dry_and_stays_in_the_denominator():
  t, x = _alternating_year()
  x[364] = np.nan  # day 365 NaN, so the filled NaN of day 101 stays NaN
  x[100] = np.nan
  _, thr, frac = cq.rolling_seeps(pd.DatetimeIndex(t), x, 3, 0.5 / 1000)
  assert np.isnan(thr[100, 0])
  np.testing.assert_allclose(frac[100, 0], 0.0)  # neighbours 99, 101 are wet
  np.testing.assert_allclose(frac[102, 0], 1 / 3)


def test_short_day_axis_repeats_slots_in_the_window():
  t = _times('2021-12-22', '2022-01-01', 24)  # day labels 356..365
  rs = np.random.RandomState(3)
  x = rs.normal(size=(t.size, 2))
  labels, got = cq.rolling_quantile(pd.DatetimeIndex(t), x, 31, [0.2, 0.5])
  assert labels.size == 10 and got.shape == (2, 10, 2)
  w = co.window_weights(31)
  for d in range(10):
    for c in range(2):  # tap j reads slot (d + j - 15) mod 10
      s = np.array([x[(d + j - 15) % 10, c] for j in range(31)])
      np.testing.assert_allclose(got[:, d, c],
                                 cq.weighted_quantile(s, w, [0.2, 0.5]),
                                 rtol=1e-14)


def test_constant_field_returns_the_constant():
  t = _times('2019-01-01', '2021-01-01', 24)
  x = np.full((t.size, 2), 7.25)
  _, got = cq.hourly_quantile(t, x, 61, slice('2019', '2020'), 24,
                              [0.0, 0.3, 1.0])
  # xarray's formula sums x * dv: exact up to the rounding of sum(dv) = 1
  np.testing.assert_allclose(got, 7.25, rtol=1e-13)


# -- the operator layer on the NumPy stand-in of the C ABI ------------------------
def make_precip(dtype=np.float32, layout='3d', nan_frac=0.0, seed=0, **kw):
  """A precipitation-like field in metres: about 40 % exact zeros."""
  from weatherbench2_b200 import xarray_lite as xl
  ds, t, x = make_obs(layout=layout, dtype=np.float64, seed=seed, **kw)
  rs = np.random.RandomState(seed + 100)
  x = np.where(rs.uniform(size=x.shape) < 0.4, 0.0, np.abs(x) * 1e-3)
  if nan_frac:
    x[rs.uniform(size=x.shape) < nan_frac] = np.nan
  x = x.astype(dtype)
  z = ds['z']
  out = xl.Dataset({'z': (z.dims, x), 'orog': (z.dims[1:], x[0])},
                   {k: c for k, c in ds.coords.items()})
  return out, t, x


QS = (0.1, 0.5, 0.9)
# (name, kind, make kwargs, frequency, hour_interval, window, via)
# via: 'climatology' (compute_climatology) or 'stat_fn' (compute_*_stat)
QUANTILE_CASES = [
    ('hourly6_quantile_4d', 'quantile', dict(layout='4d'), 'hourly', 6, 61,
     'climatology'),
    ('hourly12_quantile_3d_f64_nan', 'quantile',
     dict(dtype=np.float64, nan_frac=0.05), 'hourly', 12, 15, 'stat_fn'),
    ('daily_quantile_4d_nan', 'quantile', dict(layout='4d', nan_frac=0.05),
     'daily', None, 31, 'stat_fn'),
    ('daily_quantile_3d_f64', 'quantile', dict(dtype=np.float64), 'daily',
     None, 61, 'climatology'),
    ('hourly6_seeps_3d_nan', 'seeps', dict(nan_frac=0.05), 'hourly', 6, 61,
     'climatology'),
    ('hourly12_seeps_4d_f64', 'seeps', dict(layout='4d', dtype=np.float64),
     'hourly', 12, 15, 'stat_fn'),
    ('daily_seeps_3d', 'seeps', {}, 'daily', None, 31, 'stat_fn'),
    ('daily_seeps_4d_f64_nan', 'seeps',
     dict(layout='4d', dtype=np.float64, nan_frac=0.05), 'daily', None, 61,
     'climatology'),
]
DRY_MM = 0.25


def _oracle(kind, t, x, frequency, hour_interval, window):
  years = slice('2019', '2020')
  if kind == 'quantile':
    if frequency == 'hourly':
      labels, q = cq.hourly_quantile(t, x, window, years, hour_interval, QS)
    else:
      labels, q = cq.daily_quantile(t, x, window, years, QS)
    return labels, {'q': q}
  if frequency == 'hourly':
    labels, a, b = cq.hourly_seeps(t, x, window, years, hour_interval, DRY_MM)
  else:
    labels, a, b = cq.daily_seeps(t, x, window, years, DRY_MM)
  return labels, {'thr': a, 'frac': b}


def run_quantile_case(case, obs_transform=lambda ds: ds):
  """Runs one QUANTILE_CASES entry through weatherbench2_b200.utils and
  compares with the oracle (rtol 1e-5, atol 1e-6 max|x|)."""
  from weatherbench2_b200 import utils
  _, kind, kw, frequency, hour_interval, window, via = case
  ds, t, x = make_precip(**kw) if kind == 'seeps' else make_obs(**kw)
  obs = obs_transform(ds)
  years = slice('2019', '2020')
  if via == 'climatology':
    out = utils.compute_climatology(
        obs, frequency=frequency, hour_interval=hour_interval or 1,
        window_size=window, start_year=2019, end_year=2020,
        statistics=(kind,), quantiles=QS, seeps_dry_threshold_mm={'z': DRY_MM})
    assert set(out.keys()) == ({'z_quantile'} if kind == 'quantile' else
                               {'z_seeps_threshold', 'z_seeps_dry_fraction'})
    qname = 'z_quantile'
  else:
    fn = (utils.Quantile(list(QS)).compute if kind == 'quantile' else
          utils.SEEPSThreshold(DRY_MM, 'z').compute)
    if frequency == 'hourly':
      out = utils.compute_hourly_stat(obs, window, years, hour_interval, fn)
    else:
      out = utils.compute_daily_stat(obs, window, years, fn)
    qname = 'z'
  got = ({'q': out[qname]} if kind == 'quantile' else
         {'thr': out['z_seeps_threshold'], 'frac': out['z_seeps_dry_fraction']})
  labels, want = _oracle(kind, t, x, frequency, hour_interval, window)
  other = tuple(d for d in ds['z'].dims if d != 'time')
  lead = ('hour',) if frequency == 'hourly' else ()
  atol = 1e-6 * np.nanmax(np.abs(x))
  for key, da in got.items():
    qdim = ('quantile',) if key == 'q' else ()
    assert da.dims == lead + qdim + ('dayofyear',) + other, (key, da.dims)
    np.testing.assert_array_equal(da.coords['dayofyear'].values, labels)
    if key == 'q':
      np.testing.assert_array_equal(da.coords['quantile'].values, QS)
    vals = da.values
    assert vals.dtype == np.float32
    np.testing.assert_allclose(vals, want[key], rtol=1e-5, atol=atol,
                               err_msg=f'{case[0]} {key}')
  return got


@pytest.mark.parametrize('case', QUANTILE_CASES,
                         ids=[c[0] for c in QUANTILE_CASES])
def test_operator_layer_matches_the_oracle_on_fake_ctx(case):
  import fake_ctx_climatology_quantile
  with fake_ctx_climatology_quantile.installed() as fake:
    run_quantile_case(case)
  assert [c[0] for c in fake.calls] == ['climatology_quantile_host']


def test_error_cases():
  import fake_ctx_climatology_quantile
  from weatherbench2_b200 import utils
  ds, _, _ = make_obs(layout='3d')
  years = slice('2019', '2020')
  with fake_ctx_climatology_quantile.installed() as fake:
    for kw in (dict(statistics=('quantile',), quantiles=[0.5]),
               dict(statistics=('seeps',), seeps_dry_threshold_mm={'z': 1})):
      with pytest.raises(NotImplementedError):
        utils.compute_climatology(ds, method='fast', **kw)
    for fn in (utils.Quantile([0.5]).compute,
               utils.SEEPSThreshold(0.25, 'z').compute):
      with pytest.raises(NotImplementedError):
        utils.compute_hourly_stat_fast(ds, 61, years, 6, fn)
      with pytest.raises(NotImplementedError):
        utils.compute_daily_stat_fast(ds, 61, years, fn)
      with pytest.raises(NotImplementedError, match='out of its scope'):
        fn(ds, dim=('window', 'year'))
    for q in ([1.5], [-0.1], [0.5, np.nan]):
      with pytest.raises(ValueError):
        utils.compute_climatology(ds, statistics=('quantile',), quantiles=q,
                                  hour_interval=6)
      with pytest.raises(ValueError):
        utils.compute_hourly_stat(ds, 61, years, 6, utils.Quantile(q).compute)
    with pytest.raises(NotImplementedError, match='quantiles='):
      utils.compute_climatology(ds, statistics=('quantile',))
    with pytest.raises(NotImplementedError, match='seeps_dry_threshold_mm='):
      utils.compute_climatology(ds, statistics=('seeps',))
    # 2 stacked years x 4097 taps: beyond 8192 samples per window
    with pytest.raises(ValueError, match='8192'):
      utils.compute_hourly_stat(ds, 4097, years, 6, utils.Quantile([.5]).compute)
    with pytest.raises(KeyError):
      utils.compute_hourly_stat(ds, 61, years, 6,
                                utils.SEEPSThreshold(0.25, 'tp').compute)
    assert not fake.calls

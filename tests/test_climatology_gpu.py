"""Day-of-year climatologies through the CUDA kernels (csrc/climatology.cu)
against the float64 oracle: every operator case of test_climatology_cpu.py on
the device-tensor path and on the NumPy streamed path (a budget small enough
for many bands of cells), the float64 stress case, and a climatology built on
the GPU feeding ACC and a GaussianQuantileThreshold Brier score."""
import numpy as np
import pandas as pd
import pytest

import climatology_oracle as co
from test_climatology_cpu import OPERATOR_CASES, _times, run_operator_case

pytestmark = pytest.mark.gpu

RTOL = 1e-5


def _to_device(ds):
  import torch
  from weatherbench2_b200 import xarray_lite as xl
  out = xl.Dataset(coords=ds.coords, attrs=ds.attrs)
  for k, v in ds.items():
    out[k] = xl.DataArray(torch.from_numpy(np.ascontiguousarray(v.values)).cuda(),
                          v.dims, v.coords, k, v.attrs)
  return out


@pytest.mark.parametrize('case', OPERATOR_CASES, ids=[c[0] for c in
                                                       OPERATOR_CASES])
def test_device_tensor_path_matches_the_oracle(case):
  import torch
  got = run_operator_case(case, _to_device)
  for da in got.values():
    assert isinstance(da.data, torch.Tensor) and da.data.is_cuda


@pytest.mark.parametrize('case', OPERATOR_CASES, ids=[c[0] for c in
                                                       OPERATOR_CASES])
def test_streamed_numpy_path_in_many_bands_matches_the_oracle(case,
                                                              monkeypatch):
  from weatherbench2_b200 import _lib, utils
  # ~2 years of 6-hourly rows: about 11 KB per cell, so 64 KB of staging holds
  # two or three cells per band -- at least 7 bands, splitting latitude rows
  monkeypatch.setattr(utils, 'STREAM_BUDGET_BYTES', 64 << 10)
  ctx = _lib.default_context()
  before = ctx.launch_count
  run_operator_case(case)
  assert ctx.launch_count - before >= 5


def test_float64_moments_keep_the_std_of_a_large_mean_field():
  """1e5 + 0.5 N(0, 1) over 10 years: float32 moment sums without a shift
  lose the std entirely."""
  from weatherbench2_b200 import utils, xarray_lite as xl
  t = _times('2001-01-01', '2011-01-01', 24)
  rs = np.random.RandomState(7)
  x = (1e5 + 0.5 * rs.normal(size=(t.size, 4, 8))).astype(np.float32)
  ds = xl.Dataset({'z': (('time', 'latitude', 'longitude'), x)},
                  dict(time=t, latitude=np.arange(4.0),
                       longitude=np.arange(8.0)))
  years = slice('2001', '2010')
  _, want = co.hourly_stat(t, x.astype(np.float64), 61, years, 24, 'std')
  for obs in (ds, _to_device(ds)):
    got = utils.compute_hourly_stat(obs, 61, years, 24, 'std')['z'].values
    np.testing.assert_allclose(got, want, rtol=RTOL)
  _, want = co.hourly_stat_fast(t, x.astype(np.float64), 61, years, 24, 'std')
  got = utils.compute_hourly_stat_fast(ds, 61, years, 24, 'std')['z'].values
  np.testing.assert_allclose(got, want, rtol=RTOL)


def _oracle_climatology(truth, x, times, frequency):
  from weatherbench2_b200 import xarray_lite as xl
  years = slice('2019', '2020')
  out = xl.Dataset()
  for stat, key in (('mean', 'z'), ('std', 'z_std')):
    if frequency == 'hourly':
      labels, v = co.hourly_stat(times, x.astype(np.float64), 61, years, 6,
                                 stat)
      lead = ('hour', 'dayofyear')
    else:
      labels, v = co.daily_stat(times, x.astype(np.float64), 61, years, stat)
      lead = ('dayofyear',)
    da = truth['z']
    coords = {k: c for k, c in da.coords.items() if 'time' not in c.dims}
    coords['dayofyear'] = xl.Coord(('dayofyear',), labels)
    if frequency == 'hourly':
      coords['hour'] = xl.Coord(('hour',), np.arange(0, 24, 6))
    out[key] = xl.DataArray(v.astype(np.float32), lead + da.dims[1:], coords,
                            key)
  return out


def test_gpu_climatology_feeds_acc_and_gaussian_threshold_brier(tmp_path):
  from test_eval_probabilistic_gpu import _mock_ens
  from test_evaluation_cpu import _data_config, _forecast
  from weatherbench2_b200 import config, evaluation, metrics, thresholds
  from weatherbench2_b200 import utils, xarray_lite as xl
  # ACC and the climatology forecast through evaluate_in_memory
  t = _times('2019-01-01', '2021-01-01', 6)
  ti = pd.DatetimeIndex(t)
  rs = np.random.RandomState(0)
  lat, lon = np.linspace(-90, 90, 9), np.linspace(0, 360, 12, endpoint=False)
  season = 3 * np.sin(2 * np.pi * np.asarray(ti.dayofyear) / 365.25)
  x = (season[:, None, None, None] + rs.normal(size=(t.size, 2, 12, 9))
       ).astype(np.float32)
  dims = ('time', 'level', 'longitude', 'latitude')
  truth = xl.Dataset({'z': (dims, x)}, dict(time=t, level=np.array([500, 850]),
                                           longitude=lon, latitude=lat))
  gpu = utils.compute_climatology(truth, hour_interval=6, start_year=2019,
                                  end_year=2020, statistics=('mean', 'std'))
  ref = _oracle_climatology(truth, x, t, 'hourly')
  fc, _, _, _ = _forecast('2020-01-01', '2020-01-08', 12, [0, 6, 30], True,
                          variables=('z',))
  results = []
  for clim in (gpu, ref):
    dc = _data_config(fc, truth, str(tmp_path), True, climatology=clim,
                      variables=['z'])
    ec = {'acc': config.Eval(metrics={'acc': metrics.ACC(climatology=clim)}),
          'clim': config.Eval(metrics={'mse': metrics.MSE()},
                              evaluate_climatology=True)}
    results.append(evaluation.evaluate_in_memory(dc, ec))
  for name in ('acc', 'clim'):
    np.testing.assert_allclose(results[0][name]['z'].values,
                               results[1][name]['z'].values, rtol=1e-5,
                               atol=1e-6, err_msg=name)
  # a Brier score against a GaussianQuantileThreshold of a daily climatology
  forecast, truth_sel, _, _, _, _, _, lat2, lon2 = _mock_ens()
  td = _times('2019-01-01', '2021-01-01', 24)
  xd = rs.normal(size=(td.size, 2, lat2.size, lon2.size)).astype(np.float32)
  daily_truth = xl.Dataset(
      {'z': (('time', 'level', 'latitude', 'longitude'), xd)},
      dict(time=td, level=np.array([500, 850]), latitude=lat2,
           longitude=lon2))
  gpu = utils.compute_climatology(daily_truth, frequency='daily',
                                  start_year=2019, end_year=2020,
                                  statistics=('mean', 'std'))
  ref = _oracle_climatology(daily_truth, xd, td, 'daily')
  briers = [metrics.EnsembleBrierScore(
      [thresholds.GaussianQuantileThreshold(climatology=c, quantile=0.75)]
  ).compute(forecast, truth_sel)['z'].values for c in (gpu, ref)]
  assert np.isfinite(briers[0]).all()
  np.testing.assert_allclose(briers[0], briers[1], rtol=1e-5, atol=1e-6)

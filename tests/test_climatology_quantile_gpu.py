"""Quantile and SEEPS climatologies through the CUDA kernel
(csrc/climatology_quantile.cu) against the float64 oracle: every operator case
of test_climatology_quantile_cpu.py on device tensors and on NumPy input
streamed in many bands, a 30-year window-61 case on a sample of cells, ties
and constant fields, and GPU-built climatologies feeding the quantile-threshold
Brier score and SEEPS."""
import numpy as np
import pandas as pd
import pytest

import climatology_quantile_oracle as cq
from test_climatology_cpu import _times
from test_climatology_gpu import _to_device
from test_climatology_quantile_cpu import QUANTILE_CASES, run_quantile_case

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('case', QUANTILE_CASES,
                         ids=[c[0] for c in QUANTILE_CASES])
def test_device_tensor_path_matches_the_oracle(case):
  import torch
  got = run_quantile_case(case, _to_device)
  for da in got.values():
    assert isinstance(da.data, torch.Tensor) and da.data.is_cuda


@pytest.mark.parametrize('case', QUANTILE_CASES,
                         ids=[c[0] for c in QUANTILE_CASES])
def test_streamed_numpy_path_in_many_bands_matches_the_oracle(case,
                                                              monkeypatch):
  from weatherbench2_b200 import _lib, utils
  # ~2 years of 6-hourly rows plus the outputs: tens of KB per cell, so 64 KB
  # of staging holds one or two cells per band
  monkeypatch.setattr(utils, 'STREAM_BUDGET_BYTES', 64 << 10)
  ctx = _lib.default_context()
  before = ctx.launch_count
  run_quantile_case(case)
  assert ctx.launch_count - before >= 5


def _series(start, stop, step_h, shape, seed, kind='normal'):
  from weatherbench2_b200 import xarray_lite as xl
  t = _times(start, stop, step_h)
  rs = np.random.RandomState(seed)
  if kind == 'normal':
    x = rs.normal(size=(t.size,) + shape)
  elif kind == 'ties':  # a handful of distinct values: long runs of ties
    x = rs.randint(0, 4, size=(t.size,) + shape) * 0.5
  else:
    x = np.full((t.size,) + shape, 3.7)
  x = x.astype(np.float32)
  ds = xl.Dataset({'z': (('time', 'latitude', 'longitude'), x)},
                  dict(time=t, latitude=np.arange(shape[0], dtype=float),
                       longitude=np.arange(shape[1], dtype=float)))
  return ds, t, x


def test_thirty_years_window_61_on_a_sample_of_cells():
  from weatherbench2_b200 import utils
  ds, t, x = _series('1990-01-01', '2020-01-01', 6, (3, 16), 11)
  qs = [0.1, 0.25, 0.5, 0.75, 0.9]
  years = slice('1990', '2019')
  got = utils.compute_hourly_stat(_to_device(ds), 61, years, 6,
                                  utils.Quantile(qs).compute)['z'].values
  assert got.shape == (4, 5, 366, 3, 16)
  rs = np.random.RandomState(5)
  for i, j in zip(rs.randint(0, 3, 4), rs.randint(0, 16, 4)):
    _, want = cq.hourly_quantile(t, x[:, i, j, None], 61, years, 6, qs)
    np.testing.assert_allclose(got[..., i, j], want[..., 0], rtol=1e-5,
                               atol=1e-6 * np.abs(x).max(), err_msg=(i, j))


@pytest.mark.parametrize('kind', ['ties', 'constant'])
def test_ties_and_constant_fields(kind):
  from weatherbench2_b200 import utils
  ds, t, x = _series('2018-01-01', '2021-01-01', 12, (2, 8), 4, kind)
  qs = [0.0, 0.3, 0.5, 2 / 3, 1.0]
  years = slice('2018', '2020')
  for obs in (ds, _to_device(ds)):
    got = utils.compute_hourly_stat(obs, 31, years, 12,
                                    utils.Quantile(qs).compute)['z'].values
    if kind == 'constant':  # the constant, exactly
      np.testing.assert_array_equal(got, np.float32(3.7))
    else:
      _, want = cq.hourly_quantile(t, x, 31, years, 12, qs)
      np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-6)


def test_gpu_quantile_climatology_feeds_the_threshold_brier_score():
  from test_eval_probabilistic_gpu import _mock_ens
  from weatherbench2_b200 import metrics, thresholds, utils
  from weatherbench2_b200 import xarray_lite as xl
  forecast, truth_sel, _, _, _, _, _, lat, lon = _mock_ens()
  td = _times('2019-01-01', '2021-01-01', 24)
  rs = np.random.RandomState(2)
  xd = rs.normal(size=(td.size, 2, lat.size, lon.size)).astype(np.float32)
  dims = ('time', 'level', 'latitude', 'longitude')
  hist = xl.Dataset({'z': (dims, xd)},
                    dict(time=td, level=np.array([500, 850]), latitude=lat,
                         longitude=lon))
  qs = [0.25, 0.5, 0.75]
  gpu = utils.compute_climatology(_to_device(hist), frequency='daily',
                                  start_year=2019, end_year=2020,
                                  statistics=('quantile',), quantiles=qs)
  labels, want = cq.daily_quantile(td, xd, 61, slice('2019', '2020'), qs)
  coords = {k: c for k, c in hist['z'].coords.items() if 'time' not in c.dims}
  coords['dayofyear'] = xl.Coord(('dayofyear',), labels)
  coords['quantile'] = xl.Coord(('quantile',), np.asarray(qs))
  ref = xl.Dataset({'z_quantile': xl.DataArray(
      want.astype(np.float32), ('quantile', 'dayofyear') + dims[1:], coords,
      'z_quantile')})
  briers = [metrics.EnsembleBrierScore(
      [thresholds.QuantileThreshold(climatology=c, quantile=0.75)]
  ).compute(forecast, truth_sel)['z'].values for c in (gpu, ref)]
  assert np.isfinite(briers[0]).all()
  np.testing.assert_allclose(briers[0], briers[1], rtol=1e-5, atol=1e-6)


def test_gpu_seeps_climatology_feeds_seeps():
  from test_seeps_gpu import NAME, _pair
  from weatherbench2_b200 import evaluation, metrics, utils
  from weatherbench2_b200 import xarray_lite as xl
  fds, tds, _, truth = _pair()
  tsel = evaluation.select_truth_at_valid_time(tds, fds)
  dims, _ = truth['vars'][NAME]
  coords = {k: v for k, v in truth['coords'].items() if k != 'time'}
  other = tuple(np.asarray(coords[d]).size for d in dims if d != 'time')
  t = _times('2019-01-01', '2021-01-01', 6)
  rs = np.random.RandomState(8)
  x = np.where(rs.uniform(size=(t.size,) + other) < 0.4, 0.0,
               rs.gamma(0.8, 2e-3, size=(t.size,) + other)).astype(np.float32)
  hist = xl.Dataset({NAME: (dims, x)}, dict(coords, time=t))
  gpu = utils.compute_climatology(hist, hour_interval=6, start_year=2019,
                                  end_year=2020, statistics=('seeps',),
                                  seeps_dry_threshold_mm={NAME: 0.25})
  labels, thr, frac = cq.hourly_seeps(t, x, 61, slice('2019', '2020'), 6, 0.25)
  cc = {k: xl.Coord((k,), np.asarray(v)) for k, v in coords.items()}
  cc['dayofyear'] = xl.Coord(('dayofyear',), labels)
  cc['hour'] = xl.Coord(('hour',), np.arange(0, 24, 6))
  cdims = ('hour', 'dayofyear') + tuple(d for d in dims if d != 'time')
  ref = xl.Dataset({
      NAME + '_seeps_threshold': xl.DataArray(thr.astype(np.float32), cdims,
                                              cc),
      NAME + '_seeps_dry_fraction': xl.DataArray(frac.astype(np.float32),
                                                 cdims, cc)})
  res = [metrics.SEEPS(climatology=c).compute(fds, tsel)[NAME].values
         for c in (gpu, ref)]
  assert np.isfinite(res[0]).all()
  np.testing.assert_allclose(res[0], res[1], rtol=1e-5, atol=1e-6)
  pd.testing.assert_index_equal(pd.Index(gpu[NAME + '_seeps_threshold']
                                         .coords['dayofyear'].values),
                                pd.Index(labels))

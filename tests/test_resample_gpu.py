"""Time resampling and rolling windows through the CUDA kernels
(csrc/resample.cu) against the float64 oracle: every operator case of
test_resample_cpu.py on device tensors and on NumPy input streamed in many
bands, the C ABI directly (forecast layout read in place, float64, rolling
windows up to and past the staged limit, NaN / Inf / gaps, a 1e5 + N(0, 1)
field, every argument error), and weekly means feeding MSE on the device."""
import re

import numpy as np
import pandas as pd
import pytest

import resample_oracle as ro
from test_resample_cpu import (ALIGNED_CASES, OPERATOR_CASES, aligned_case,
                               assert_matches, check_aligned,
                               run_operator_case)

pytestmark = pytest.mark.gpu


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
  from weatherbench2_b200 import _lib, resampling
  # at most 60 steps and 3 statistics of 8 B per cell: 4 KB of staging holds
  # one or two cells per band, so every variable takes many bands
  monkeypatch.setattr(resampling, 'STREAM_BUDGET_BYTES', 4 << 10)
  ctx = _lib.default_context()
  before = ctx.launch_count
  run_operator_case(case)
  assert ctx.launch_count - before >= 5


@pytest.mark.parametrize('case', ALIGNED_CASES, ids=str)
def test_resample_equals_rolling_on_common_times(case):
  """Rolling sums slide (add the entering step, subtract the leaving one),
  so the two agree to float64 rounding rather than bit for bit."""
  res, roll, _ = aligned_case(case)
  check_aligned(res, roll, rtol=1e-14)


def _series(shape, dtype, seed, nan_inf=True, offset=0.0):
  rs = np.random.RandomState(seed)
  x = offset + rs.normal(size=shape)
  if nan_inf:
    flat = x.reshape(-1)
    n = flat.size
    flat[rs.choice(n, n // 97, replace=False)] = np.nan
    flat[rs.choice(n, n // 211, replace=False)] = np.inf
    flat[rs.choice(n, n // 223, replace=False)] = -np.inf
  return x.astype(dtype)


def _device_call(x, bins=None, window=0, skipna=False, stats=ro.STATISTICS,
                 axis=1):
  """wb2_time_window_stats on x (device, read in place along `axis`)."""
  import torch
  from weatherbench2_b200 import _lib
  ctx = _lib.default_context()
  xt = torch.from_numpy(x).cuda()
  shape = x.shape
  nouter, ntime = int(np.prod(shape[:axis])), shape[axis]
  ninner = int(np.prod(shape[axis + 1:]))
  start, count = bins if bins is not None else (None, None)
  nout = ntime if window else len(count)
  oshape = shape[:axis] + (nout,) + shape[axis + 1:]
  out = {s: torch.empty(oshape, dtype=xt.dtype, device='cuda') for s in stats}
  ctx.time_window_stats(xt.data_ptr(), _lib.F64 if x.dtype == np.float64 else
                        _lib.F32, nouter, ntime, ninner, start, count, window,
                        skipna, *(out[s].data_ptr() if s in out else None
                                  for s in ro.STATISTICS))
  return {s: v.cpu().numpy() for s, v in out.items()}


@pytest.mark.parametrize('dtype', [np.float32, np.float64])
@pytest.mark.parametrize('window', [1, 7, 28, 120, 168, 200])
def test_rolling_windows_with_nan_and_inf(window, dtype):
  """Outer 2 x 700 steps (three output blocks) x 37 inner cells (a partial
  CTA); 168 is the staged limit, 200 takes the direct path."""
  x = _series((2, 700, 37), dtype, window)
  want = ro.rolling(x, window, axis=1)
  got = _device_call(x, window=window)
  for s in ro.STATISTICS:
    assert_matches(got[s], want[s], s, x, 1)
  got = _device_call(x, window=window, stats=('mean',))  # sum-only staging
  assert_matches(got['mean'], want['mean'], 'mean', x, 1)


@pytest.mark.parametrize('dtype', [np.float32, np.float64])
@pytest.mark.parametrize('skipna', [False, True])
def test_resample_with_gaps_nan_and_inf(skipna, dtype):
  rs = np.random.RandomState(3)
  count = rs.randint(0, 9, size=150).astype(np.int32)
  count[[0, 5, 6, 149]] = 0
  ntime = int(count.sum()) + 4
  start = np.cumsum(count) - count + 2  # two leading and trailing steps unused
  x = _series((3, ntime, 50), dtype, 4)
  x[1, :, 7] = np.nan  # an all-NaN cell
  want = ro.resample(x, start, count, skipna=skipna, axis=1)
  got = _device_call(x, (start, count), skipna=skipna)
  for s in ro.STATISTICS:
    assert_matches(got[s], want[s], s, x, 1)


def test_forecast_layout_is_read_in_place_along_prediction_timedelta():
  """(time, prediction_timedelta, level, longitude, latitude) float64,
  weekly bins over 28 daily leads: the series address is the tensor's own."""
  x = _series((5, 28, 3, 24, 13), np.float64, 6, nan_inf=False)
  start, count = np.arange(0, 28, 7), np.full(4, 7, np.int32)
  want = ro.resample(x, start, count, axis=1)
  got = _device_call(x, (start, count))
  for s in ro.STATISTICS:
    assert_matches(got[s], want[s], s, x, 1)


def test_large_mean_field_keeps_mean_and_sum_precision():
  """1e5 + N(0, 1): float64 accumulation keeps mean and sum to float32
  rounding, for daily bins of 6-hourly data and a 28-step rolling window."""
  x = _series((1, 2000, 300), np.float32, 8, nan_inf=False, offset=1e5)
  start, count = np.arange(0, 2000, 4), np.full(500, 4, np.int32)
  want = ro.resample(x, start, count, ('mean', 'sum'), axis=1)
  got = _device_call(x, (start, count), stats=('mean', 'sum'))
  for s in ('mean', 'sum'):
    assert_matches(got[s], want[s], s, x, 1)
  want = ro.rolling(x, 28, ('mean', 'sum'), axis=1)
  got = _device_call(x, window=28, stats=('mean', 'sum'))
  for s in ('mean', 'sum'):
    assert_matches(got[s], want[s], s, x, 1)


def test_argument_errors_launch_nothing():
  import torch
  from weatherbench2_b200 import _lib
  ctx = _lib.default_context()
  x = torch.zeros((2, 10, 4), device='cuda')
  out = torch.empty((2, 10, 4), device='cuda')
  xh = np.zeros((2, 10, 4), np.float32)
  oh = np.empty((2, 10, 4), np.float32)
  s3, c3 = np.array([0, 3, 6]), np.array([3, 3, 3])
  o = out.data_ptr()
  bad = [  # (message fragment, dtype, ntime, start, count, window, outputs)
      ('dtype', 7, 10, s3, c3, 0, (o, None, None, None)),
      ('exactly one', _lib.F32, 10, s3, c3, 3, (o, None, None, None)),
      ('exactly one', _lib.F32, 10, None, None, 0, (o, None, None, None)),
      ('both be given', _lib.F32, 10, s3, None, 0, (o, None, None, None)),
      ('window must be >= 0', _lib.F32, 10, None, None, -2,
       (o, None, None, None)),
      ('none of mean', _lib.F32, 10, s3, c3, 0, (None, None, None, None)),
      ('bin_count[1]', _lib.F32, 10, s3, np.array([3, -1, 3]), 0,
       (None, o, None, None)),
      ('bin_start[2]', _lib.F32, 10, np.array([0, 3, 11]),
       np.array([3, 3, 0]), 0, (None, None, o, None)),
      ('bin_start[0]', _lib.F32, 10, np.array([-1, 3, 6]), c3, 0,
       (None, None, None, o)),
      ('ends past ntime', _lib.F32, 10, np.array([0, 3, 8]), c3, 0,
       (o, None, None, None)),
      ('overlaps', _lib.F32, 10, np.array([0, 2, 6]), c3, 0,
       (o, None, None, None)),
      ('overlaps', _lib.F32, 10, np.array([3, 0, 6]), c3, 0,
       (o, None, None, None)),
      ('ntime / ninner', _lib.F32, -1, None, None, 3, (o, None, None, None)),
  ]
  before = ctx.launch_count
  for msg, dtype, ntime, start, count, window, outs in bad:
    with pytest.raises(_lib.Wb2Error, match=re.escape(msg)):
      ctx.time_window_stats(x.data_ptr(), dtype, 2, ntime, 4, start, count,
                            window, False, *outs)
    host_outs = tuple(oh.ctypes.data if p else None for p in outs)
    with pytest.raises(_lib.Wb2Error, match=re.escape(msg)):
      ctx.time_window_stats_host(xh.ctypes.data, dtype, 2, ntime, 4, start,
                                 count, window, False, 1 << 20, *host_outs)
  ctx.synchronize()
  assert ctx.launch_count == before


def test_weekly_means_on_the_device_feed_mse():
  """Weekly means of a GPU-resident forecast along prediction_timedelta and
  of the truth at the same valid times feed MSE().compute_chunk as CUDA
  tensors; the MSE matches the one of the oracle's weekly means."""
  import torch
  from weatherbench2_b200 import metrics, resampling, xarray_lite as xl
  rs = np.random.RandomState(9)
  lat, lon = np.linspace(-90, 90, 33), np.arange(0, 360, 5.625)
  lead = pd.timedelta_range('0 day', '13 days', freq='1D').values
  times = pd.date_range('2020-01-01', periods=4).values
  dims = ('time', 'prediction_timedelta', 'latitude', 'longitude')
  coords = dict(time=times, prediction_timedelta=lead, latitude=lat,
                longitude=lon)
  shape = (times.size, lead.size, lat.size, lon.size)
  f = rs.normal(size=shape).astype(np.float32)
  t = (f + rs.normal(size=shape)).astype(np.float32)
  weekly = {}
  for name, v in (('forecast', f), ('truth', t)):
    ds = xl.Dataset({'z': (dims, torch.from_numpy(v).cuda())}, coords)
    weekly[name] = resampling.resample_in_time(
        ds, period='7D', mean_vars=['z'], time_dim='prediction_timedelta')
    assert weekly[name]['z'].data.is_cuda
  got = metrics.MSE().compute_chunk(weekly['forecast'], weekly['truth'])['z']
  start, count = np.array([0, 7]), np.array([7, 7], np.int32)
  ref = {}
  wcoords = dict(coords, prediction_timedelta=lead[[0, 7]])
  for name, v in (('forecast', f), ('truth', t)):
    m = ro.resample(v, start, count, ['mean'], axis=1)['mean'].astype(
        np.float32)
    ref[name] = xl.Dataset({'z': (dims, m)}, wcoords)
  want = metrics.MSE().compute_chunk(ref['forecast'], ref['truth'])['z']
  assert np.isfinite(got.values).all()
  np.testing.assert_allclose(got.values, want.values, rtol=2e-6)

"""GPU tests of wb2_precip_accumulation / wb2_precip_accumulation_host
(csrc/precip_accumulation.cu) and the precipitation derived variables
(weatherbench2/derived_variables.py:471-528, 685-720): every output bit-equal
to tests/precip_oracle.py, NaN positions and the sign of zero included, for
torch CUDA input and for NumPy input streamed in many bands; 721 x 1440
fields, one inner cell, inner counts off the 128-byte tile, a 1000-step lead
axis whose windows straddle CTA blocks, windows 1 .. the staged cap and past
the series, float64; a window whose sum depends on its order; every argument
error of the entries; the aggregate against the rolling sum it is; and both
inside the metric loop with MSE and SEEPS."""
import numpy as np
import pytest

import precip_oracle as po

pytestmark = pytest.mark.gpu

LEAD = 'prediction_timedelta'
CAP = 1024


def _assert_bits(got, want, what):
  got, want = np.asarray(got), np.asarray(want)
  assert got.dtype == want.dtype, (what, got.dtype, want.dtype)
  assert got.shape == want.shape, what
  np.testing.assert_array_equal(np.isnan(got), np.isnan(want), err_msg=what)
  u = np.uint32 if got.dtype == np.float32 else np.uint64
  same = (got.view(u) == want.view(u)) | np.isnan(want)
  if not same.all():
    i = tuple(np.argwhere(~same)[0])
    raise AssertionError(f'{what}: {(~same).sum()} values differ, first at {i}: '
                         f'{got[i]!r} vs {want[i]!r}')


def _series(nouter, ntime, ninner, dtype, seed, specials=True):
  """Cumulative precipitation with negative steps, NaN, +-Inf and signed
  zeros: [nouter][ntime][ninner]."""
  rs = np.random.RandomState(seed)
  steps = rs.exponential(1e-3, size=(nouter, ntime, ninner))
  steps[rs.uniform(size=steps.shape) < 0.2] *= -0.1
  x = np.cumsum(steps, axis=1).astype(dtype)
  if specials and x.size > 64:
    flat = x.reshape(-1)
    pick = rs.choice(flat.size, size=min(40, flat.size // 8), replace=False)
    vals = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0], dtype)
    flat[pick] = vals[np.arange(pick.size) % vals.size]
    if ninner > 1:  # a cell that sits at zero, with -0.0 steps
      x[:, :, -1] = 0.0
      x[:, 1::3, -1] = -0.0
  return x


def _run(ctx, x, window, clamp=True, budget=None):
  """(device result, host-streamed result) of one entry call each."""
  import torch
  from weatherbench2_b200 import _lib
  nouter, ntime, ninner = x.shape
  code = _lib.F32 if x.dtype == np.float32 else _lib.F64
  xd = torch.from_numpy(x).cuda()
  od = torch.empty_like(xd)
  ctx.precip_accumulation(xd.data_ptr(), code, nouter, ntime, ninner, window,
                          clamp, od.data_ptr())
  oh = np.full_like(x, 7.0)
  per_cell = 2 * ntime * x.itemsize
  ctx.precip_accumulation_host(
      x.ctypes.data, code, nouter, ntime, ninner, window, clamp,
      budget if budget is not None else 2 * per_cell * 5, oh.ctypes.data)
  ctx.synchronize()
  return od.cpu().numpy(), oh


CASES = {
    # name: (nouter, ntime, ninner, dtype, windows)
    'ninner1_ntime1000': (3, 1000, 1, np.float32, (1, 4, 24, 999, 1000, 1500)),
    'ninner37_ntime1100_cap': (2, 1100, 37, np.float32, (4, 255, 256, CAP)),
    'ninner45_f64': (3, 300, 45, np.float64, (1, 6, 24, 299, 300, 2000)),
    'ninner100_short': (5, 41, 100, np.float32, (1, 4, 40, 41)),
}


@pytest.mark.parametrize('case', sorted(CASES))
def test_device_and_streamed_bit_equal_to_the_oracle(case):
  from weatherbench2_b200 import _lib
  ctx = _lib.default_context()
  nouter, ntime, ninner, dtype, windows = CASES[case]
  x = _series(nouter, ntime, ninner, dtype, seed=len(case))
  for w in windows:
    for clamp in (True, False):
      want = po.accumulate(x, w, clamp, axis=1)
      dev, host = _run(ctx, x, w, clamp)
      _assert_bits(dev, want, f'{case} w={w} clamp={clamp} device')
      _assert_bits(host, want, f'{case} w={w} clamp={clamp} host')
  # bands of whole outer indices, the last one partial
  per_cell = 2 * ntime * x.itemsize
  budget = 2 * per_cell * ninner * 2
  want = po.accumulate(x, 4, True, axis=1)
  _, host = _run(ctx, x, 4, True, budget=budget)
  _assert_bits(host, want, f'{case} outer bands')


def test_full_size_fields_through_the_derived_variable():
  """(2 inits, 41 six-hourly leads, 721 x 1440) and the dictionary entry:
  a CUDA tensor in, a CUDA tensor of the same dtype out."""
  import torch
  from weatherbench2_b200 import derived_variables as dv, xarray_lite as xl
  x = _series(2, 41, 721 * 1440, np.float32, seed=11).reshape(2, 41, 721, 1440)
  lead = (np.arange(41) * 6).astype('timedelta64[h]').astype('timedelta64[ns]')
  coords = {'time': np.arange(2), LEAD: lead,
            'latitude': np.linspace(-90, 90, 721),
            'longitude': np.arange(1440) * 0.25}
  dims = ('time', LEAD, 'latitude', 'longitude')
  want = po.accumulate(x, 4, True, axis=1)
  dev = xl.Dataset({'total_precipitation': (dims, torch.from_numpy(x).cuda())},
                   coords)
  got = dv.DERIVED_VARIABLE_DICT['total_precipitation_24hr'].compute(dev)
  assert got.dims == dims and got.data.is_cuda
  assert got.data.dtype == torch.float32
  _assert_bits(got.data.cpu().numpy(), want, '721x1440 device')
  host = xl.Dataset({'total_precipitation': (dims, x)}, coords)
  got = dv.DERIVED_VARIABLE_DICT['total_precipitation_24hr'].compute(host)
  assert isinstance(got.values, np.ndarray)
  _assert_bits(got.values, want, '721x1440 host')
  np.testing.assert_array_equal(got.coords[LEAD].values, lead)


def test_window_summed_oldest_first():
  from weatherbench2_b200 import _lib
  ctx = _lib.default_context()
  for dtype in (np.float32, np.float64):
    x = np.array([0, 2.0**60, 0, 1], dtype).reshape(1, 4, 1)
    dev, host = _run(ctx, x, 3)
    assert dev[0, 3, 0] == 1 and host[0, 3, 0] == 1  # newest first gives 0
    assert np.isnan(dev[0, :3]).all() and np.isnan(host[0, :3]).all()


def test_every_argument_error_and_one_launch_per_call():
  import torch
  from weatherbench2_b200 import _lib
  ctx = _lib.default_context()
  x = torch.zeros((2, 1500, 3), device='cuda')
  out = torch.empty_like(x)
  xh = np.zeros((2, 1500, 3), np.float32)
  oh = np.empty_like(xh)
  good = dict(x=x.data_ptr(), dtype=_lib.F32, nouter=2, ntime=1500, ninner=3,
              window=4, clamp_negative=True, out=out.data_ptr())
  goodh = dict(good, x=xh.ctypes.data, out=oh.ctypes.data, budget=1 << 20)
  bad = [dict(dtype=2), dict(dtype=-1), dict(nouter=-1), dict(ntime=-1),
         dict(ninner=-1), dict(window=0), dict(window=-3),
         dict(window=CAP + 1), dict(window=1499),
         dict(x=None), dict(out=None),
         dict(nouter=0, ninner=0, ntime=65535 * 256 + 1),
         dict(nouter=1 << 31, ninner=1, ntime=1)]
  for change in bad:
    with pytest.raises(_lib.Wb2Error):
      ctx.precip_accumulation(**dict(good, **change))
    with pytest.raises(_lib.Wb2Error):
      ctx.precip_accumulation_host(**dict(goodh, **change))
  ctx.synchronize()
  before = ctx.launch_count
  ctx.precip_accumulation(**good)
  ctx.precip_accumulation(**dict(good, window=CAP))
  ctx.precip_accumulation(**dict(good, ntime=600, window=600))  # staged, all NaN
  ctx.precip_accumulation(**dict(good, window=1500))   # past the cap: all NaN
  ctx.synchronize()
  assert ctx.launch_count - before == 4
  assert torch.isnan(out).all()
  ctx.precip_accumulation(**dict(good, nouter=0))       # nothing to do
  ctx.precip_accumulation(**dict(good, ninner=0))
  ctx.precip_accumulation_host(**dict(goodh, ntime=0))
  ctx.synchronize()
  assert ctx.launch_count - before == 4


@pytest.mark.parametrize('on_device', [True, False])
def test_aggregate_is_the_rolling_sum(on_device):
  import torch
  from weatherbench2_b200 import derived_variables as dv, resampling
  from weatherbench2_b200 import xarray_lite as xl
  rs = np.random.RandomState(4)
  acc = rs.exponential(1e-3, size=(3, 41, 57, 33)).astype(np.float32)
  acc[0, 5, 3, 2] = np.nan
  acc[1, 9, 0, 0] = np.inf
  dims = ('time', 'lead_time', 'latitude', 'longitude')
  lead = (np.arange(41) * 6).astype('timedelta64[h]').astype('timedelta64[ns]')
  data = torch.from_numpy(acc).cuda() if on_device else acc
  ds = xl.Dataset({'total_precipitation_6hr': (dims, data)},
                  {'lead_time': lead, 'time': np.arange(3)})
  got = dv.AggregatePrecipitationAccumulation(
      24, lead_time_name='lead_time').compute(ds)
  want = resampling.resample_in_time_core(
      ds, 'rolling', '24h', 'sum', False, time_dim='lead_time')
  g = got.data.cpu().numpy() if on_device else got.values
  w = want['total_precipitation_6hr']
  w = w.data.cpu().numpy() if on_device else w.values
  assert got.dims == dims
  _assert_bits(g, w, 'aggregate')
  assert np.isnan(g[:, :3]).all()


def _metric_loop_inputs(on_device):
  import torch
  import wb2_testdata as td
  from weatherbench2_b200 import evaluation, xarray_lite as xl
  kw = dict(variables_3d=[], variables_2d=['total_precipitation'],
            time_start='2020-01-01', time_stop='2020-01-04',
            spatial_resolution_in_degrees=30)
  fc = td.mock_forecast_data(lead_stop='2 day', lead_resolution='6 hours',
                             **kw)
  tr = td.mock_truth_data(**dict(kw, time_stop='2020-01-07'),
                          time_resolution='6 hours')
  rs = np.random.RandomState(8)
  d, v = fc['vars']['total_precipitation']
  steps = rs.exponential(1e-3, size=v.shape)
  steps[rs.uniform(size=v.shape) < 0.1] *= -0.2
  fc['vars']['total_precipitation'] = (d, np.cumsum(steps, axis=0).astype(
      np.float32))
  d, v = tr['vars']['total_precipitation']
  tr['vars']['total_precipitation'] = (d, np.cumsum(
      rs.exponential(1e-3, size=v.shape), axis=0).astype(np.float32))
  mk = lambda p: xl.Dataset({k: dv_ for k, dv_ in p['vars'].items()},  # noqa: E731
                            p['coords'])
  fds = evaluation.apply_time_conventions(mk(fc), by_init=True)
  tds = evaluation.select_truth_at_valid_time(mk(tr), fds)
  if on_device:
    f = fds['total_precipitation']
    fds['total_precipitation'] = xl.DataArray(
        torch.from_numpy(np.ascontiguousarray(f.values)).cuda(), f.dims,
        dict(f.coords))
  return fds, tds


def _seeps_climatology(tds):
  from weatherbench2_b200 import xarray_lite as xl
  rs = np.random.RandomState(9)
  t = tds['total_precipitation']
  lon = t.coords['longitude'].values
  lat = t.coords['latitude'].values
  shape = (4, 366, lon.size, lat.size)
  cdims = ('hour', 'dayofyear', 'longitude', 'latitude')
  name = 'total_precipitation_24hr'
  return xl.Dataset(
      {name + '_seeps_dry_fraction': (cdims, rs.uniform(
          0.05, 0.9, size=shape).astype(np.float32)),
       name + '_seeps_threshold': (cdims, rs.uniform(
           5e-4, 4e-3, size=shape).astype(np.float32))},
      {'hour': np.array([0, 6, 12, 18]), 'dayofyear': np.arange(1, 367),
       'longitude': lon, 'latitude': lat})


@pytest.mark.parametrize('on_device', [True, False])
def test_metric_loop_with_mse_and_seeps(on_device):
  """Truth lazily gathered at the valid times, forecast on the device or in
  host memory: the derived variable gives the same bits as the oracle's
  accumulations fed in as variables.  MSE reads forecast and truth from one
  memory space, so it runs on the host forecast; SEEPS runs on both."""
  import torch
  from weatherbench2_b200 import config, derived_variables as dv, evaluation
  from weatherbench2_b200 import metrics, xarray_lite as xl
  fds, tds = _metric_loop_inputs(on_device)
  clim = _seeps_climatology(tds)
  name = 'total_precipitation_24hr'
  mets = {'seeps': metrics.SEEPS(climatology=clim)}
  if not on_device:
    mets['mse'] = metrics.MSE()
  var = dv.PrecipitationAccumulation('total_precipitation', 24,
                                     lead_time_name='lead_time')
  ec = config.Eval(metrics=mets, derived_variables={name: var})
  got = evaluation._metric_and_region_loop(fds, tds, ec, skipna=False)  # pylint: disable=protected-access

  fds2, tds2 = _metric_loop_inputs(on_device)
  f = fds2['total_precipitation']
  li = f.dims.index('lead_time')
  fv = f.data.cpu().numpy() if on_device else np.asarray(f.values)
  # C-contiguous like the entry's output, so the metric kernels see the same
  # layout and reduce in the same order
  facc = np.ascontiguousarray(po.accumulate(fv, 4, True, axis=li))
  fds2[name] = xl.DataArray(torch.from_numpy(facc).cuda() if on_device
                            else facc, f.dims, dict(f.coords))
  t = tds2['total_precipitation']
  tacc = np.ascontiguousarray(po.accumulate(
      np.asarray(t.values), 4, True, axis=t.dims.index('lead_time')))
  tds2[name] = xl.DataArray(tacc, t.dims, dict(t.coords))
  ec2 = config.Eval(metrics=mets, derived_variables={})
  want = evaluation._metric_and_region_loop(fds2, tds2, ec2, skipna=False)  # pylint: disable=protected-access

  assert sorted(got.keys()) == sorted(want.keys())
  assert name in got.keys()
  for k in got.keys():
    g, w = got[k], want[k]
    assert g.dims == w.dims, k
    gv = g.data.cpu().numpy() if hasattr(g.data, 'cpu') else np.asarray(g.values)
    wv = w.data.cpu().numpy() if hasattr(w.data, 'cpu') else np.asarray(w.values)
    _assert_bits(gv, wv, k)
  seeps = np.asarray(want[name].values)
  assert np.isfinite(seeps).any()

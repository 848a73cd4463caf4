"""The launch layer of the metric operators (`_spatial.run_*`) on the NumPy
stand-in context (tests/fake_ctx.py): every device buffer a metric call
allocates -- staged uploads of host operands, region-group outputs, map
outputs -- is freed when the call returns, when a check rejects the staged
operands and when the kernel itself fails; a truth operand that carries the
ensemble dimension is rejected with `ValueError` on the K2, ensemble-map,
threshold and rank-histogram paths."""
import numpy as np
import pytest

import fake_ctx
import wb2_testdata as td

T2M = '2m_temperature'
PRECIP = 'total_precipitation_24hr'


def _ds(vars, coords):  # pylint: disable=redefined-builtin
  from weatherbench2_b200 import xarray_lite as xl
  return xl.Dataset({k: (d, v) for k, (d, v) in vars.items()}, coords)


def _cast(ds, dtype):
  return {'vars': {k: (d, v.astype(dtype)) for k, (d, v) in ds['vars'].items()},
          'coords': ds['coords']}


def _pair(ensemble_size=None, dtype=np.float32, variables=('geopotential',)):
  truth, forecast = td.get_random_truth_and_forecast(
      variables=variables, ensemble_size=ensemble_size, lead_stop='1 day',
      time_stop='2019-12-02', time_resolution='12 hours')
  return (_ds(**_cast(forecast, dtype)), _ds(**_cast(truth, dtype)))


def _land(fds):
  from weatherbench2_b200 import regions
  lat, lon = fds['latitude'].values, fds['longitude'].values
  lsm = np.random.RandomState(0).rand(lat.size, lon.size)
  lsm[lsm < 0.3] = 0.0
  return regions.LandRegion(lsm)


def _climatology(fds):
  """(dayofyear, level, longitude, latitude) climatology of geopotential."""
  lat, lon = fds['latitude'].values, fds['longitude'].values
  clim = np.random.RandomState(9).normal(
      size=(366, 3, lon.size, lat.size)).astype(np.float32)
  return _ds({'geopotential': (('dayofyear', 'level', 'longitude',
                                'latitude'), clim)},
             {'dayofyear': 1 + np.arange(366), 'level': np.array([850, 500,
                                                                  700]),
              'latitude': lat, 'longitude': lon})


def _threshold_case(kind):
  """Ensemble forecast of 2m temperature and thresholds of `kind`."""
  from weatherbench2_b200 import thresholds
  kw = dict(variables_3d=[], variables_2d=[T2M], time_start='2022-01-01',
            time_stop='2022-01-02', spatial_resolution_in_degrees=30)
  rs = np.random.RandomState(3)
  forecast = td.mock_forecast_data(ensemble_size=3, lead_stop='1 day', **kw)
  truth = td.mock_truth_data(**kw)
  for ds in (forecast, truth):
    for k, (d, v) in ds['vars'].items():
      ds['vars'][k] = (d, rs.normal(size=v.shape).astype(np.float32))
  dims, arr = truth['vars'][T2M]
  first = np.take(arr, 0, axis=dims.index('time'))
  sdims = tuple(d for d in dims if d != 'time')
  coords = {k: v for k, v in truth['coords'].items() if k != 'time'}
  coords['dayofyear'] = np.arange(1, 367)
  rep = np.broadcast_to(first, (366,) + first.shape).copy()
  if kind == 'gaussian':
    clim = _ds({T2M: (('dayofyear',) + sdims, rep),
                T2M + '_std': (('dayofyear',) + sdims, rep + 1.0)}, coords)
    thrs = [thresholds.GaussianQuantileThreshold(climatology=clim, quantile=q)
            for q in (0.2, 0.7)]
  else:
    coords['quantile'] = np.array([0.2, 0.7])
    clim = _ds({T2M + '_quantile': (('quantile', 'dayofyear') + sdims,
                                    np.stack([rep - 0.5, rep + 0.5]))}, coords)
    thrs = [thresholds.QuantileThreshold(climatology=clim, quantile=q)
            for q in (0.2, 0.7)]
  return _ds(**forecast), _ds(**truth), thrs


def _gaussian_case():
  kw = dict(variables_3d=[], variables_2d=[T2M, T2M + '_std'],
            time_start='2022-01-01', time_stop='2022-01-02',
            spatial_resolution_in_degrees=30)
  forecast = td.random_like(td.mock_forecast_data(lead_stop='1 day', **kw), 4)
  d, v = forecast['vars'][T2M + '_std']
  forecast['vars'][T2M + '_std'] = (d, np.abs(v) + 0.1)
  truth = td.random_like(td.mock_truth_data(
      variables_3d=[], variables_2d=[T2M], time_start='2022-01-01',
      time_stop='2022-01-05', spatial_resolution_in_degrees=30), 5)
  return _ds(**_cast(forecast, np.float32)), _ds(**_cast(truth, np.float32))


def _seeps_case():
  from weatherbench2_b200 import evaluation
  kw = dict(variables_3d=[], variables_2d=[PRECIP], time_start='2022-01-01',
            time_stop='2022-01-04', spatial_resolution_in_degrees=30)
  rs = np.random.RandomState(12)
  forecast = td.mock_forecast_data(lead_stop='1 day', **kw)
  truth = td.mock_truth_data(**dict(kw, time_stop='2022-01-06'))
  for ds in (forecast, truth):
    d, v = ds['vars'][PRECIP]
    ds['vars'][PRECIP] = (d, rs.gamma(0.6, 0.002, v.shape).astype(np.float32))
  fds = evaluation.apply_time_conventions(_ds(**forecast), by_init=True)
  tds = evaluation.select_truth_at_valid_time(_ds(**truth), fds)
  dims, arr = truth['vars'][PRECIP]
  sdims = tuple(d for d in dims if d != 'time')
  shape = (4, 366) + tuple(arr.shape[dims.index(d)] for d in sdims)
  coords = {k: v for k, v in truth['coords'].items() if k != 'time'}
  coords['hour'] = np.array([0, 6, 12, 18])
  coords['dayofyear'] = np.arange(1, 367)
  cdims = ('hour', 'dayofyear') + sdims
  clim = _ds({PRECIP + '_seeps_dry_fraction':
                  (cdims, rs.uniform(0, 1, shape).astype(np.float32)),
              PRECIP + '_seeps_threshold':
                  (cdims, rs.uniform(5e-4, 4e-3, shape).astype(np.float32))},
             coords)
  return fds, tds, clim


def _mse_with_climatology():
  from weatherbench2_b200 import metrics
  fds, tds = _pair()
  regions = [None, _land(fds)]
  clim = _climatology(fds)

  def call():
    with metrics.batch(regions=regions, climatology=clim):
      metrics.MSE().compute_chunk(fds, tds, region=regions[1])
      metrics.ACC(climatology=clim).compute_chunk(fds, tds, region=regions[0])
  return call


def _wind_vector():
  from weatherbench2_b200 import metrics
  u, v = 'u_component_of_wind', 'v_component_of_wind'
  fds, tds = _pair(variables=(u, v))
  metric = metrics.WindVectorMSE(u_name=u, v_name=v, vector_name='wv')
  return lambda: metric.compute_chunk(fds, tds, region=_land(fds))


def _crps():
  from weatherbench2_b200 import metrics
  fds, tds = _pair(ensemble_size=3)
  regions = [None, _land(fds)]

  def call():
    with metrics.batch(regions=regions):
      metrics.CRPS().compute_chunk(fds, tds, region=regions[1])
  return call


def _energy_score():
  from weatherbench2_b200 import metrics
  fds, tds = _pair(ensemble_size=3)
  return lambda: metrics.EnergyScore().compute_chunk(fds, tds,
                                                     region=_land(fds))


def _spatial_mse():
  from weatherbench2_b200 import metrics
  fds, tds = _pair()
  return lambda: metrics.SpatialMSE().compute(fds, tds)


def _spatial_crps():
  from weatherbench2_b200 import metrics
  fds, tds = _pair(ensemble_size=3)
  return lambda: metrics.SpatialCRPS().compute(fds, tds)


def _brier(kind):
  def make():
    from weatherbench2_b200 import metrics
    fds, tds, thrs = _threshold_case(kind)
    return lambda: metrics.EnsembleBrierScore(thrs).compute_chunk(
        fds, tds, region=_land(fds))
  return make


def _gaussian_crps():
  from weatherbench2_b200 import metrics
  fds, tds = _gaussian_case()
  return lambda: metrics.GaussianCRPS().compute_chunk(fds, tds,
                                                      region=_land(fds))


def _spatial_brier():
  from weatherbench2_b200 import metrics
  fds, tds, thrs = _threshold_case('field')
  return lambda: metrics.SpatialEnsembleBrierScore(thrs).compute(fds, tds)


def _spatial_seeps():
  from weatherbench2_b200 import metrics
  fds, tds, clim = _seeps_case()
  return lambda: metrics.SpatialSEEPS(climatology=clim).compute(fds, tds)


def _rank_histogram():
  from weatherbench2_b200 import metrics
  fds, tds = _pair(ensemble_size=3)
  return lambda: metrics.RankHistogram(seed=1).compute(fds, tds)


FAMILIES = {
    'mse_acc_climatology': _mse_with_climatology,
    'wind_vector_mse': _wind_vector,
    'crps_host_entry': _crps,
    'energy_score_k3': _energy_score,
    'spatial_mse': _spatial_mse,
    'spatial_crps': _spatial_crps,
    'brier_field_thresholds': _brier('field'),
    'brier_gaussian_thresholds': _brier('gaussian'),
    'gaussian_crps': _gaussian_crps,
    'spatial_brier': _spatial_brier,
    'spatial_seeps': _spatial_seeps,
    'rank_histogram': _rank_histogram,
}


@pytest.mark.parametrize('family', sorted(FAMILIES))
def test_nothing_outlives_a_call(family):
  """A second call leaves as many live buffers as the first: staged uploads
  and outputs are freed.  The first call may leave the land-mask cells, which
  the context caches."""
  with fake_ctx.installed() as fake:
    call = FAMILIES[family]()
    call()
    after_first = len(fake._bufs)  # pylint: disable=protected-access
    calls_first = len(fake.calls)
    call()
    assert len(fake._bufs) == after_first  # pylint: disable=protected-access
    assert len(fake.calls) == 2 * calls_first > 0


class KernelFailure(RuntimeError):
  pass


class FailingContext(fake_ctx.FakeContext):
  """A stand-in whose kernel entries raise: the launch layer has staged the
  inputs and allocated the outputs by then."""
  failures = 0


def _fail(self, *args, **kwargs):
  del args, kwargs
  self.failures += 1
  raise KernelFailure('kernel failed')


for _entry in ('det_metrics', 'det_metrics_vector', 'ens_metrics',
               'ens_metrics_host', 'energy_score', 'det_maps', 'ens_maps',
               'ens_threshold_metrics', 'ens_threshold_maps',
               'gaussian_metrics', 'seeps_maps', 'rank_histogram'):
  setattr(FailingContext, _entry, _fail)


@pytest.mark.parametrize('family', sorted(FAMILIES))
def test_nothing_outlives_a_failed_kernel(family):
  """Only the cached land-mask cells stay allocated after a kernel raised."""
  with fake_ctx.installed(FailingContext) as fake:
    call = FAMILIES[family]()
    with pytest.raises(KernelFailure):
      call()
    assert fake.failures == 1
    cells = set(fake.__dict__.get('_cell_weight_cache', {}).values())
    assert set(fake._bufs) == cells  # pylint: disable=protected-access


def _staged_launches():
  """Direct launches whose operands are uploaded before the launch fails:
  `_check_grid` rejects a float64 operand, and the K2 staging branch (taken
  when not every operand is float32 on the host) meets a failing kernel."""
  from weatherbench2_b200 import _lib, _spatial as sp
  fds, tds = _pair()
  f = sp.prepare_operand(fds['geopotential'], None, np.float32)
  t64 = sp.prepare_operand(tds['geopotential'], f.layout, np.float64)
  xds, xtds, _ = _threshold_case('field')
  x = sp.prepare_operand(xds[T2M], None, np.float32)
  t = sp.prepare_operand(xtds[T2M], x.layout, np.float32)
  x64 = sp.prepare_operand(xds[T2M], None, np.float64)
  thr64 = sp.prepare_operand(xtds[T2M], x.layout, np.float64)
  lat, lon = xds['latitude'].values, xds['longitude'].values
  ens = 'realization'
  return {
      'det_maps_mixed_dtypes': (ValueError, lambda ctx: sp.run_det_maps(
          ctx, f, t64, _lib.MAP_MSE, None, False)),
      'ens_maps_float64': (ValueError, lambda ctx: sp.run_ens_maps(
          ctx, x64, t, ens, _lib.ENS_CRPS, None, False)),
      'threshold_stats_float64_field': (
          ValueError, lambda ctx: sp.run_ens_threshold_metrics(
              ctx, x, t, ens, ('field', [thr64]), lat, lon, [None], False)),
      'k2_staged_kernel_failure': (
          KernelFailure, lambda ctx: sp.run_ens_metrics(
              ctx, [x64], [t], ens, lat, lon, [None], False)),
  }


@pytest.mark.parametrize('case', ['det_maps_mixed_dtypes', 'ens_maps_float64',
                                  'threshold_stats_float64_field',
                                  'k2_staged_kernel_failure'])
def test_staged_uploads_are_freed_when_the_launch_raises(case):
  with fake_ctx.installed(FailingContext) as fake:
    error, launch = _staged_launches()[case]
    with pytest.raises(error):
      launch(fake)
    assert fake.h2d_bytes > 0  # the operands were uploaded
    assert not fake._bufs  # pylint: disable=protected-access


def _truth_with_members():
  """An ensemble pair whose first variable has a valid truth and whose second
  variable's truth has the ensemble dimension."""
  from weatherbench2_b200 import xarray_lite as xl
  fds, tds = _pair(ensemble_size=3, variables=('geopotential', 'temperature'))
  bad = xl.Dataset({'geopotential': tds['geopotential'],
                    'temperature': fds['temperature']})
  return fds, bad


# EnergyScore's K3 path does not check the truth's dimensions.
def _rejections():
  from weatherbench2_b200 import metrics
  fds, tds = _truth_with_members()
  ffds, _, thrs = _threshold_case('field')
  return {
      'k2': lambda: metrics.CRPS().compute_chunk(fds, tds),
      'ens_maps': lambda: metrics.SpatialCRPS().compute(fds, tds),
      'threshold_stats': lambda: metrics.EnsembleBrierScore(
          thrs).compute_chunk(ffds, ffds),
      'threshold_maps': lambda: metrics.SpatialEnsembleBrierScore(
          thrs).compute(ffds, ffds),
      'rank_histogram': lambda: metrics.RankHistogram(seed=1).compute(
          fds, tds),
  }


@pytest.mark.parametrize('path', ['k2', 'ens_maps', 'threshold_stats',
                                  'threshold_maps', 'rank_histogram'])
def test_truth_with_ensemble_dim_is_rejected(path):
  """`ValueError`, and the call leaves no buffer behind (the map paths have
  run the first variable by then)."""
  with fake_ctx.installed() as fake:
    call = _rejections()[path]
    with pytest.raises(ValueError, match='realization'):
      call()
    assert not fake._bufs  # pylint: disable=protected-access

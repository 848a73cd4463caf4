"""The xarray boundary of the public operators (xarray_lite.boundary), driven
on the NumPy stand-in contexts (tests/fake_ctx*.py) with the stand-in `xarray`
package (tests/fake_xarray):

  (a) every operator family called with native xarray arguments returns a
      native object that converts back to exactly what the lite call returns;
  (b) every Metric, DerivedVariable and Threshold subclass of the package has
      its public methods behind the boundary;
  (c) a native call converts each native argument once;
  (d) no module but xarray_lite converts between the two, except the
      evaluation writers, which hand a lite result to xarray's netCDF / zarr
      writers."""
import collections
import importlib
import os
import re
import sys

import numpy as np
import pandas as pd
import pytest

import fake_ctx
import fake_ctx_average
import fake_ctx_climatology_quantile
import fake_ctx_column
import fake_ctx_dynamics
import fake_ctx_precip
import fake_ctx_quantile
import fake_ctx_reindex
import fake_ctx_resample
import fake_ctx_thermo
import test_climatology_cpu as clim_cases
import test_metric_launch_cpu as launch
import test_reindex_cpu as reindex_cases

HERE = os.path.dirname(os.path.abspath(__file__))
FAKE = os.path.join(HERE, 'fake_xarray')
PKG = os.path.join(HERE, '..', 'weatherbench2_b200')


@pytest.fixture
def xr(monkeypatch):
  monkeypatch.syspath_prepend(FAKE)
  sys.modules.pop('xarray', None)
  mod = importlib.import_module('xarray')
  assert mod.__version__ == '0.0-fake'
  yield mod
  sys.modules.pop('xarray', None)


def _xl():
  from weatherbench2_b200 import xarray_lite as xl
  return xl


def _same_values(got, want):
  got, want = np.asarray(got), np.asarray(want)
  assert got.dtype == want.dtype and got.shape == want.shape
  if got.dtype.kind in 'biufcmM':
    assert got.tobytes() == want.tobytes()  # bit for bit, NaNs included
  else:
    assert np.array_equal(got, want)


def _same_coords(got: dict, want: dict):
  assert set(got) == set(want)
  for k, c in want.items():
    assert got[k].dims == c.dims and got[k].attrs == c.attrs, k
    _same_values(got[k].values, c.values)


def _same_array(got, want):
  assert type(got).__name__ == 'DataArray'
  assert (got.dims, got.name, got.attrs) == (want.dims, want.name, want.attrs)
  _same_values(got.values, want.values)
  _same_coords(got.coords, want.coords)


def _same(got, want):
  xl = _xl()
  if isinstance(want, xl.DataArray):
    _same_array(got, want)
    return
  assert isinstance(got, xl.Dataset)
  assert set(got.keys()) == set(want.keys()) and got.attrs == want.attrs
  for k in want.keys():
    _same_array(got[k], want[k])
  _same_coords(got.coords, want.coords)


def _native(obj):
  xl = _xl()
  return xl.to_xarray(obj) if isinstance(obj, (xl.Dataset, xl.DataArray)) else (
      obj)


def _check(xr, installed, fn, *args, **kwargs):
  """`fn` on lite arguments, then on the same arguments converted to native
  xarray: the native call returns the native kind of the lite result, which
  converts back to it exactly.  Returns the lite result."""
  xl = _xl()
  native_args = [_native(a) for a in args]
  native_kwargs = {k: _native(v) for k, v in kwargs.items()}
  with installed():
    lite = fn(*args, **kwargs)
    native = fn(*native_args, **native_kwargs)
  assert isinstance(lite, (xl.Dataset, xl.DataArray))
  assert isinstance(native, xr.Dataset if isinstance(lite, xl.Dataset)
                    else xr.DataArray)
  _same(xl.from_xarray(native), lite)
  return lite


# -- (a) every family, natively -------------------------------------------------
def _metric_cases():
  from weatherbench2_b200 import metrics
  fds, tds = launch._pair()  # pylint: disable=protected-access
  xds, xtds = launch._pair(ensemble_size=3)  # pylint: disable=protected-access
  gds, gtds, thrs = launch._threshold_case('gaussian')  # pylint: disable=protected-access
  sds, stds, sclim = launch._seeps_case()  # pylint: disable=protected-access
  return [(metrics.MSE(), fds, tds), (metrics.CRPS(), xds, xtds),
          (metrics.EnsembleBrierScore(thrs), gds, gtds),
          (metrics.SEEPS(climatology=sclim), sds, stds),
          (metrics.RankHistogram(seed=3), xds, xtds)]


@pytest.mark.parametrize('index', range(5))
@pytest.mark.parametrize('method', ['compute_chunk', 'compute'])
def test_metric_families(xr, index, method):
  metric, forecast, truth = _metric_cases()[index]
  got = _check(xr, fake_ctx.installed, getattr(metric, method), forecast,
               truth)
  if method == 'compute' and index in (1, 4):
    assert got.attrs['ensemble_size'] == 3


def test_lat_weights_and_central_reliability(xr):
  from weatherbench2_b200 import metrics
  fds, tds = launch._pair(ensemble_size=3)  # pylint: disable=protected-access
  _check(xr, fake_ctx.installed, metrics.get_lat_weights, fds)
  with fake_ctx.installed():
    hist = metrics.RankHistogram(seed=3).compute(fds, tds)
  _check(xr, fake_ctx.installed, metrics.central_reliability, hist)
  got = _check(xr, fake_ctx.installed, metrics.central_reliability,
               hist['geopotential'])
  assert got.name == 'geopotential'


def test_threshold_compute(xr):
  _, tds, gaussian = launch._threshold_case('gaussian')  # pylint: disable=protected-access
  _, _, quantile = launch._threshold_case('field')  # pylint: disable=protected-access
  for thr in (gaussian[0], quantile[0]):
    _check(xr, fake_ctx.installed, thr.compute, tds)


def _atmosphere(nlat=6, nlon=8):
  """(time, level, latitude, longitude) float32 fields of every derived
  variable's inputs, latitudes off the poles."""
  xl = _xl()
  rs = np.random.RandomState(4)
  dims = ('time', 'level', 'latitude', 'longitude')
  shape = (2, 3, nlat, nlon)
  lat = np.linspace(-75, 75, nlat)
  lon = np.arange(nlon) * 360.0 / nlon
  level = np.array([500.0, 700.0, 850.0])
  fields = {
      'u_component_of_wind': rs.normal(size=shape),
      'v_component_of_wind': rs.normal(size=shape),
      'temperature': 250 + 10 * rs.uniform(size=shape),
      'geopotential': (9.81 * (6000 - 5 * level)[:, None, None]
                       + rs.normal(size=shape)),
      'specific_humidity': rs.uniform(1e-4, 1e-2, size=shape)}
  coords = {'time': np.array(['2020-01-01', '2020-01-02'], 'datetime64[ns]'),
            'level': level, 'latitude': lat, 'longitude': lon}
  return xl.Dataset({k: (dims, v.astype(np.float32))
                     for k, v in fields.items()}, coords)


def _precipitation():
  xl = _xl()
  rs = np.random.RandomState(5)
  dims = ('time', 'prediction_timedelta', 'latitude', 'longitude')
  tp = np.cumsum(rs.gamma(0.6, 0.002, (2, 5, 3, 4)), axis=1)
  coords = {'time': np.array(['2020-01-01', '2020-01-02'], 'datetime64[ns]'),
            'prediction_timedelta': np.arange(5) * np.timedelta64(6, 'h'),
            'latitude': np.array([-30.0, 0.0, 30.0]),
            'longitude': np.arange(4) * 90.0}
  return xl.Dataset({'total_precipitation': (dims, tp.astype(np.float32)),
                     'total_precipitation_6hr': (dims,
                                                 tp.astype(np.float32))},
                    coords)


def test_derived_variable_modules(xr):
  from weatherbench2_b200 import derived_variables as dvs
  ds = _atmosphere()
  wind = dvs.WindSpeed(u_name='u_component_of_wind',
                       v_name='v_component_of_wind')
  got = _check(xr, fake_ctx_dynamics.installed, wind.compute, ds)
  assert got.name is None  # np.sqrt(u**2 + v**2) of the reference
  _check(xr, fake_ctx_dynamics.installed, dvs.WindDivergence().compute, ds)
  _check(xr, fake_ctx_column.installed, dvs.TotalColumnWater().compute, ds)
  _check(xr, fake_ctx_thermo.installed, dvs.LapseRate().compute, ds)
  _check(xr, fake_ctx_thermo.installed, dvs.RelativeHumidity().compute, ds)
  precip = _precipitation()
  for dv in (dvs.PrecipitationAccumulation(
      total_precipitation_name='total_precipitation', accumulation_hours=12),
             dvs.AggregatePrecipitationAccumulation(accumulation_hours=12)):
    got = _check(xr, fake_ctx_precip.installed, dv.compute, precip)
    assert got.name == dv.base_variables[0]


def test_zonal_spectrum_and_interpolation(xr):
  from weatherbench2_b200 import derived_variables as dvs
  ds = _atmosphere()
  spectrum = dvs.ZonalEnergySpectrum('u_component_of_wind')
  got = _check(xr, fake_ctx.installed, spectrum.compute, ds)
  assert got.name == 'u_component_of_wind'
  _check(xr, fake_ctx.installed, spectrum.compute_latitude_mean, ds,
         time_mean_dim='time')
  _check(xr, fake_ctx.installed, dvs.interpolate_spectral_frequencies, got,
         'zonal_wavenumber')


def test_regridding(xr):
  from weatherbench2_b200 import regridding as rg
  ds = _atmosphere(nlat=19, nlon=36)[['temperature']]
  src = rg.Grid.from_degrees(ds['longitude'].values, ds['latitude'].values)
  tgt = rg.Grid.from_degrees(np.linspace(0, 360, 12, endpoint=False),
                             np.linspace(-60, 60, 7))
  regridder = rg.ConservativeRegridder(src, tgt)
  _check(xr, fake_ctx.installed, regridder.regrid_dataset,
         ds.transpose('time', 'level', 'longitude', 'latitude'))


def test_preprocessing(xr):
  from weatherbench2_b200 import preprocessing as pp
  ds = _atmosphere()[['temperature', 'specific_humidity']]
  members = ds.expand_dims({'realization': 3})
  _check(xr, fake_ctx.installed, pp.compute_ensemble_mean, members)
  _check(xr, fake_ctx_quantile.installed, pp.compute_quantiles_core, ds,
         [0.25, 0.5], 'time')
  _check(xr, fake_ctx_quantile.installed, pp.compute_quantiles, ds,
         [0.25, 0.5], ['time', 'longitude'])
  _check(xr, fake_ctx_average.installed, pp.compute_averages, ds,
         ['latitude', 'longitude'])
  _check(xr, fake_ctx_average.installed, pp.moment_reduce, ds, 'second')
  _check(xr, fake_ctx_average.installed, pp.compute_statistical_moments, ds)


def test_resampling(xr):
  from weatherbench2_b200 import resampling
  ds, _, _ = clim_cases.make_obs(layout='3d', start='2020-01-01',
                                 stop='2020-01-10')
  _check(xr, fake_ctx_resample.installed, resampling.resample_in_time_core,
         ds, 'resample', '1D', 'mean', False)
  _check(xr, fake_ctx_resample.installed, resampling.resample_in_time_core,
         ds['z'], 'rolling', '1D', 'max', False)
  _check(xr, fake_ctx_resample.installed, resampling.resample_in_time, ds,
         period='1D', mean_vars=['ALL'], max_vars=['z'])


@pytest.mark.parametrize('statistics', [('mean', 'std'), ('quantile',)])
def test_climatology(xr, statistics):
  from weatherbench2_b200 import utils
  ds, _, _ = clim_cases.make_obs(layout='3d')
  _check(xr, fake_ctx_climatology_quantile.installed, utils.compute_climatology,
         ds, frequency='daily', window_size=5, start_year=2019, end_year=2020,
         statistics=statistics, quantiles=[0.5])


def test_reindexing(xr):
  from weatherbench2_b200 import reindexing as ri
  V = reindex_cases.V  # pylint: disable=invalid-name
  forecast = reindex_cases._ivt_input(  # pylint: disable=protected-access
      V['ivt|no_offset_delta|x'].astype(np.float32),
      V['ivt|no_offset_delta|lead_hours'])
  _check(xr, fake_ctx_reindex.installed, ri.index_on_valid_time, forecast)
  clim, _ = reindex_cases._climatology(reindex_cases.CLIM_DIMS[0])  # pylint: disable=protected-access
  _check(xr, fake_ctx_reindex.installed, ri.expand_climatology, clim,
         time_start='2020-01-01', time_stop='2020-01-03')
  truth, _, _ = reindex_cases._truth()  # pylint: disable=protected-access
  _check(xr, fake_ctx_reindex.installed,
         ri.compute_probabilistic_climatological_forecasts, truth,
         **reindex_cases.PROB_KW)
  sampled = np.array([['1991-01-02', '1991-01-04'], ['1991-01-03', '1991-01-01']],
                     'datetime64[ns]')
  _check(xr, fake_ctx_reindex.installed, ri.sample_forecasts_core, truth,
         sampled, pd.to_datetime(['1992-01-01', '1992-01-02']),
         pd.to_timedelta(['0h', '6h']))


def test_evaluation_loop(xr):
  from weatherbench2_b200 import config, evaluation, metrics
  fds, tds = launch._pair()  # pylint: disable=protected-access
  eval_config = config.Eval(metrics={'mse': metrics.MSE(),
                                     'bias': metrics.Bias()})
  _check(xr, fake_ctx.installed, evaluation._metric_and_region_loop, fds,  # pylint: disable=protected-access
         tds, eval_config, False, compute_chunk=True)


# -- (b) no subclass left out ------------------------------------------------------
def _subclasses(cls):
  for sub in cls.__subclasses__():
    yield sub
    yield from _subclasses(sub)


def test_every_public_method_is_behind_the_boundary():
  from weatherbench2_b200 import derived_variables, metrics, thresholds
  xl = _xl()
  wrapper = xl.boundary(lambda: None).__code__
  families = [(metrics.Metric, ('compute', 'compute_chunk')),
              (derived_variables.DerivedVariable, ('compute',
                                                   'compute_latitude_mean')),
              (thresholds.Threshold, ('compute',))]
  seen = 0
  for base, names in families:
    for cls in [base, *_subclasses(base)]:
      assert cls.__module__.startswith('weatherbench2_b200'), cls
      for name in names:
        method = getattr(cls, name, None)
        if method is None:
          continue
        assert method.__code__ is wrapper, f'{cls.__name__}.{name}'
        seen += 1
  assert seen > 100  # every metric, derived variable and threshold class


# -- (c) one conversion per call -------------------------------------------------
def _count_conversions(monkeypatch):
  xl = _xl()
  counts = collections.Counter()
  convert = xl.from_xarray

  def counting(obj):
    if xl.is_native_xarray(obj):
      counts[id(obj)] += 1
    return convert(obj)

  monkeypatch.setattr(xl, 'from_xarray', counting)
  return counts


def test_climatology_converts_its_input_once(xr, monkeypatch):
  from weatherbench2_b200 import utils
  ds, _, _ = clim_cases.make_obs(layout='3d')
  obs = _native(ds)
  counts = _count_conversions(monkeypatch)
  with fake_ctx_climatology_quantile.installed():
    utils.compute_climatology(obs, frequency='daily', window_size=5,
                              start_year=2019, end_year=2020,
                              statistics=('mean', 'std', 'quantile'),
                              quantiles=[0.5])
  assert counts == {id(obs): 1}


@pytest.mark.parametrize('ensemble_size', [None, 3])
def test_metric_compute_converts_each_input_once(xr, monkeypatch,
                                                 ensemble_size):
  from weatherbench2_b200 import metrics
  fds, tds = launch._pair(ensemble_size=ensemble_size)  # pylint: disable=protected-access
  forecast, truth = _native(fds), _native(tds)
  metric = metrics.MSE() if ensemble_size is None else metrics.CRPS()
  counts = _count_conversions(monkeypatch)
  with fake_ctx.installed():
    metric.compute(forecast, truth)
  assert counts == {id(forecast): 1, id(truth): 1}


# -- (d) conversion lives in one module --------------------------------------------
def test_only_xarray_lite_converts():
  found = []
  for fn in sorted(os.listdir(PKG)):
    if not fn.endswith('.py') or fn == 'xarray_lite.py':
      continue
    with open(os.path.join(PKG, fn)) as f:
      for n, line in enumerate(f, 1):
        if not re.search(r'\b(is_native_xarray|to_xarray)\(', line):
          continue
        # the evaluation writers hand the lite result to xarray's writers
        if fn == 'evaluation.py' and re.search(r'\.to_(netcdf|zarr)\(', line):
          continue
        found.append(f'{fn}:{n}: {line.strip()}')
  assert not found, '\n'.join(found)

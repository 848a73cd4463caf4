"""The rule that sends the streamed operators' NumPy input to the `*_host`
entries (weatherbench2_b200/_streamed.py), on the NumPy stand-ins of the
entries, for each family: quantiles, averages, time resampling, precipitation
accumulation, the mean and quantile climatologies, the zonal spectrum (per
time, time sum, latitude mean with and without a time mean) and conservative
regridding.

  * input already in the entry's layout and dtype reaches the entry in place,
    with no host copy;
  * float64 or transposed spectrum and regrid input reaches the entry as a
    contiguous float32 copy, with the same result;
  * the streaming budget is the module constant's value when the operator is
    called, so that a caller (or a test forcing many bands) can change it;
  * a climatology variable without cells, and a spectrum or regrid variable
    without fields, gives empty float32 results without calling the entry."""
import inspect

import numpy as np
import pandas as pd
import pytest

import fake_ctx
import fake_ctx_average
import fake_ctx_climatology
import fake_ctx_climatology_quantile
import fake_ctx_precip
import fake_ctx_quantile
import fake_ctx_resample
from test_climatology_cpu import _times, make_obs
from weatherbench2_b200 import _derived_precip
from weatherbench2_b200 import derived_variables
from weatherbench2_b200 import preprocessing as pp
from weatherbench2_b200 import regridding
from weatherbench2_b200 import resampling
from weatherbench2_b200 import utils
from weatherbench2_b200 import xarray_lite as xl

YEARS = slice('2019', '2020')


def _field(shape):
  return np.random.RandomState(0).standard_normal(shape).astype(np.float32)


def _quantile():
  x = _field((4, 6, 5))
  ds = xl.Dataset({'t': (('time', 'lat', 'lon'), x)})
  return x, lambda: pp.compute_quantiles_core(ds, [0.25, 0.5], 'lat')


def _average():
  x = _field((4, 6, 5))
  ds = xl.Dataset({'t': (('time', 'latitude', 'longitude'), x)})
  return x, lambda: pp.moment_reduce(ds, 'first')


def _resample():
  x = _field((6, 3))
  ds = xl.Dataset({'t': (('time', 'lat'), x)},
                  {'time': pd.date_range('2020-01-01', periods=6).values})
  return x, lambda: resampling.resample_in_time_core(ds, 'resample', '2D',
                                                     'mean', False)


def _precip():
  lead = 'prediction_timedelta'
  x = np.cumsum(np.abs(_field((2, 5))), axis=1, dtype=np.float32)
  ds = xl.Dataset({'tp': (('time', lead), x)},
                  {lead: np.arange(5) * np.timedelta64(6, 'h')})
  op = _derived_precip.PrecipitationAccumulation('tp', 12, lead)
  return x, lambda: op.compute(ds)


def _climatology():
  ds, _, _ = make_obs(layout='3d')
  return ds['z'].data, lambda: utils.compute_hourly_stat(ds, 61, YEARS, 6)


def _climatology_quantile():
  ds, _, _ = make_obs(layout='3d')
  fn = utils.Quantile([0.5]).compute
  return ds['z'].data, lambda: utils.compute_hourly_stat(ds, 61, YEARS, 6, fn)


# family: (its stand-in context, entry, module and name of its budget, case)
FAMILIES = {
    'quantile': (fake_ctx_quantile, 'quantile',
                 (pp, 'QUANTILE_STREAM_BUDGET_BYTES'), _quantile),
    'average': (fake_ctx_average, 'average',
                (pp, 'AVERAGE_STREAM_BUDGET_BYTES'), _average),
    'resample': (fake_ctx_resample, 'time_window_stats',
                 (resampling, 'STREAM_BUDGET_BYTES'), _resample),
    'precip': (fake_ctx_precip, 'precip_accumulation',
               (resampling, 'STREAM_BUDGET_BYTES'), _precip),
    'climatology': (fake_ctx_climatology, 'climatology',
                    (utils, 'STREAM_BUDGET_BYTES'), _climatology),
    'climatology_quantile': (fake_ctx_climatology_quantile,
                             'climatology_quantile',
                             (utils, 'STREAM_BUDGET_BYTES'),
                             _climatology_quantile),
}


def _host_calls(family):
  """Runs the family's case on its stand-in context; the arguments of every
  call of the host entry, by parameter name."""
  fakes, entry, _, case = FAMILIES[family]
  x, run = case()
  calls = []
  with fakes.installed() as fake:
    method = getattr(fake, entry + '_host')
    sig = inspect.signature(method)

    def spy(*args, **kwargs):
      calls.append(sig.bind(*args, **kwargs).arguments)
      return method(*args, **kwargs)

    setattr(fake, entry + '_host', spy)
    run()
  return x, calls


@pytest.mark.parametrize('family', FAMILIES)
def test_host_entry_reads_the_input_in_place(family):
  x, calls = _host_calls(family)
  assert x.dtype == np.float32 and x.flags.c_contiguous
  assert [c['x'] for c in calls] == [x.ctypes.data]


@pytest.mark.parametrize('family', FAMILIES)
def test_host_entry_gets_the_budget_at_call_time(family, monkeypatch):
  module, name = FAMILIES[family][2]
  monkeypatch.setattr(module, name, 3 << 20)
  _, calls = _host_calls(family)
  assert [c['budget'] for c in calls] == [3 << 20]


@pytest.mark.parametrize('quantiles', [None, [0.25, 0.75]])
def test_a_climatology_without_cells_calls_no_entry(quantiles):
  t = _times('2019-01-01', '2021-01-01', 6)
  ds = xl.Dataset({'z': (('time', 'latitude'), np.zeros((t.size, 0),
                                                         np.float32))},
                  {'time': t})
  fakes = fake_ctx_climatology_quantile  # the mean entries too
  with fakes.installed() as fake:
    if quantiles is None:
      out = utils.compute_hourly_stat(ds, 61, YEARS, 6)
      daily = utils.compute_daily_stat(ds, 61, YEARS)
      shape, dshape = (4, 366, 0), (366, 0)
    else:
      fn = utils.Quantile(quantiles).compute
      out = utils.compute_hourly_stat(ds, 61, YEARS, 6, fn)
      daily = utils.compute_daily_stat(ds, 61, YEARS, fn)
      shape, dshape = (4, 2, 366, 0), (2, 366, 0)
  assert fake.calls == []
  for got, want in ((out, shape), (daily, dshape)):
    v = got['z'].values
    assert v.dtype == np.float32 and v.shape == want



# ---- the entry pairs the zonal spectrum and conservative regridder place ----
# (`_streamed.place`): each case makes the operator's call on an input that is
# already in its host entry's layout, (time, level, latitude, longitude) for
# the spectrum and (time, level, longitude, latitude) for the regridder.
LAT, LON = np.linspace(-90, 90, 5), np.arange(8) * 45.0


def _spectrum(method, **kw):
  def make(x):
    dims = ('time', 'level', 'latitude', 'longitude')
    ds = xl.Dataset({'u': (dims, x)},
                    {'latitude': LAT, 'longitude': LON,
                     'time': np.arange(x.shape[0]),
                     'level': np.arange(x.shape[1])})
    op = derived_variables.ZonalEnergySpectrum('u')
    return lambda: getattr(op, method)(ds, **kw)
  return make


def _regrid(x):
  r = regridding.ConservativeRegridder(
      regridding.Grid.from_degrees(LON, LAT),
      regridding.Grid.from_degrees(np.arange(4) * 90.0, LAT[::2]))
  return lambda: r.regrid_array(x)


# case: (its call on an input, the host entry, the input's shape)
PLACED = {
    'spectrum': (_spectrum('compute'), 'zonal_spectrum_host', (3, 2, 5, 8)),
    'spectrum_time_sum': (_spectrum('compute', time_sum_dim='time'),
                          'zonal_spectrum_host', (3, 2, 5, 8)),
    'latitude_mean': (_spectrum('compute_latitude_mean'),
                      'zonal_spectrum_latsum_host', (3, 2, 5, 8)),
    'latitude_mean_time_mean': (
        _spectrum('compute_latitude_mean', time_mean_dim='time'),
        'zonal_spectrum_latsum_host', (3, 2, 5, 8)),
    'regrid': (_regrid, 'regrid_conservative_host', (3, 2, 8, 5)),
}


def _placed_calls(case, x):
  """Runs `case` on `x` on the stand-in context: its result, the address
  and float32 contents of the input at every call of the host entry, and
  every entry call."""
  make, entry, _ = PLACED[case]
  run = make(x)
  seen = []
  with fake_ctx.installed() as fake:
    method = getattr(fake, entry)

    def spy(addr, *args):
      seen.append((addr, fake_ctx._view(addr, x.size, np.float32).copy()))  # pylint: disable=protected-access
      return method(addr, *args)

    setattr(fake, entry, spy)
    got = run()
  return got, seen, fake.calls


@pytest.mark.parametrize('case', PLACED)
def test_placed_host_entry_reads_the_input_in_place(case):
  x = _field(PLACED[case][2])
  _, seen, _ = _placed_calls(case, x)
  assert [addr for addr, _ in seen] == [x.ctypes.data]


@pytest.mark.parametrize('layout', ['float64', 'transposed'])
@pytest.mark.parametrize('case', PLACED)
def test_placed_host_entry_gets_a_contiguous_float32_copy(case, layout):
  x = _field(PLACED[case][2])
  want, _, _ = _placed_calls(case, x)
  y = x.astype(np.float64) if layout == 'float64' else np.asfortranarray(x)
  got, seen, _ = _placed_calls(case, y)
  (addr, data), = seen
  assert addr != y.ctypes.data
  np.testing.assert_array_equal(data, x.reshape(-1))
  np.testing.assert_array_equal(np.asarray(getattr(got, 'values', got)),
                                np.asarray(getattr(want, 'values', want)))


# case: (input shape, result shape, dims, coords); None for a bare array
EMPTY = {
    'spectrum': ((0, 2, 5, 8), (0, 2, 5, 5),
                 ('time', 'level', 'latitude', 'zonal_wavenumber'),
                 {'time', 'level', 'latitude', 'zonal_wavenumber', 'frequency',
                  'wavelength'}),
    'spectrum_time_sum': ((3, 0, 5, 8), (0, 5, 5),
                          ('level', 'latitude', 'zonal_wavenumber'),
                          {'level', 'latitude', 'zonal_wavenumber',
                           'frequency', 'wavelength'}),
    'latitude_mean': ((0, 2, 5, 8), (0, 2, 5),
                      ('time', 'level', 'zonal_wavenumber'),
                      {'time', 'level', 'zonal_wavenumber'}),
    'latitude_mean_time_mean': ((3, 0, 5, 8), (0, 5),
                                ('level', 'zonal_wavenumber'),
                                {'level', 'zonal_wavenumber'}),
    'regrid': ((3, 0, 8, 5), (3, 0, 4, 3), None, None),
}


@pytest.mark.parametrize('case', EMPTY)
def test_a_variable_without_fields_calls_no_placed_entry(case):
  shape, want_shape, dims, coords = EMPTY[case]
  got, _, calls = _placed_calls(case, np.zeros(shape, np.float32))
  assert calls == []
  v = got if dims is None else got.values
  assert isinstance(v, np.ndarray)
  assert v.dtype == np.float32 and v.shape == want_shape
  if dims is not None:
    assert got.dims == dims and set(got.coords) == coords

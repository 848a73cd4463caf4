"""The rule that runs the device-only operators on whole arrays
(weatherbench2_b200/_streamed.py, `run_whole`), on the NumPy stand-ins of
their entries, for each family: wind speed, a wind-dynamics kind, total column
water, integrated vapour transport, lapse rate, relative humidity, ensemble
mean, spectrum interpolation and a bilinear regrid.

  * a second call leaves as many live device buffers as the first;
  * an entry that raises leaves no device buffer behind;
  * a variable without cells calls no entry and gives an empty result of the
    right shape and dtype.

`FAMILIES` also feeds tests/test_whole_dispatch_gpu.py."""
import numpy as np
import pytest

import fake_ctx
import fake_ctx_column
import fake_ctx_dynamics
import fake_ctx_thermo

T, Z, Q = 'temperature', 'geopotential', 'specific_humidity'
U, V = 'u_component_of_wind', 'v_component_of_wind'
DIMS = ('time', 'level', 'latitude', 'longitude')
LEVEL = np.array([300, 500, 700, 850])
LAT, LON = np.linspace(-80, 80, 9), np.arange(12) * 30.0


def _numpy(name, a):
  del name
  return a


def _atmosphere(ntime, wrap):
  """Temperature, geopotential, specific humidity and wind of realistic
  magnitude on (time, level, latitude, longitude), each passed through
  `wrap(name, array)`."""
  from weatherbench2_b200 import xarray_lite as xl
  rs = np.random.RandomState(ntime)
  shape = (ntime, LEVEL.size, LAT.size, LON.size)
  h = (44330.8 * (1 - (LEVEL / 1013.25) ** 0.190263))[:, None, None]
  f = {T: 288.15 - 6.5e-3 * h + rs.normal(scale=3, size=shape),
       Z: 9.81 * h + rs.normal(scale=40, size=shape),
       Q: np.abs(rs.normal(scale=6e-3, size=shape)) * np.exp(-h / 2500),
       U: 5 + rs.normal(scale=12, size=shape),
       V: rs.normal(scale=8, size=shape)}
  return xl.Dataset(
      {k: (DIMS, wrap(k, a.astype(np.float32))) for k, a in f.items()},
      {'time': np.arange(ntime), 'level': LEVEL, 'latitude': LAT,
       'longitude': LON})


def _derived(variable):
  def make(ntime, wrap):
    ds = _atmosphere(ntime, wrap)
    return lambda: variable().compute(ds).data
  return make


def _ensemble_mean(ntime, wrap):
  from weatherbench2_b200 import preprocessing as pp, xarray_lite as xl
  x = np.random.RandomState(1).normal(
      size=(3, ntime, LAT.size, LON.size)).astype(np.float32)
  ds = xl.Dataset({U: (('realization', 'time', 'latitude', 'longitude'),
                       wrap(U, x))})
  return lambda: pp.compute_ensemble_mean(ds)[U].data


def _spectrum_interpolation(ntime, wrap):
  from weatherbench2_b200 import derived_variables as dv, xarray_lite as xl
  nk = LON.size // 2 + 1
  spacing = np.cos(np.deg2rad(LAT)) * 2 * np.pi * dv.EARTH_RADIUS_M / LON.size
  freq = np.arange(nk)[:, None] / LON.size / spacing[None, :]
  x = np.abs(np.random.RandomState(2).normal(
      size=(ntime, LAT.size, nk))).astype(np.float32)
  spec = xl.DataArray(
      wrap(U, x), ('time', 'latitude', 'zonal_wavenumber'),
      {'latitude': xl.Coord(('latitude',), LAT),
       'frequency': xl.Coord(('zonal_wavenumber', 'latitude'), freq)})
  return lambda: dv.interpolate_spectral_frequencies(
      spec, 'zonal_wavenumber').data


def _bilinear_regrid(ntime, wrap):
  from weatherbench2_b200 import regridding as rg
  source = rg.Grid.from_degrees(np.arange(36) * 10.0, np.linspace(-90, 90, 19))
  target = rg.Grid.from_degrees(LON, LAT)
  x = np.random.RandomState(3).normal(size=(ntime, 36, 19)).astype(np.float32)
  field = wrap(U, x)
  return lambda: rg.BilinearRegridder(source, target).regrid_array(field)


def _families():
  from weatherbench2_b200 import derived_variables as dv
  # family: (the entry it calls, its operands in the operator's order, case)
  return {
      'wind_speed': ('wind_speed', (U, V),
                     _derived(lambda: dv.WindSpeed(U, V))),
      'wind_divergence': ('wind_dynamics', (U, V),
                          _derived(dv.WindDivergence)),
      'total_column_water': ('column_integral', (Q,),
                             _derived(dv.TotalColumnWater)),
      'integrated_vapor_transport': ('column_integral', (Q, U, V),
                                     _derived(dv.IntegratedWaterTransport)),
      'lapse_rate': ('lapse_rate', (T, Z), _derived(dv.LapseRate)),
      'relative_humidity': ('relative_humidity', (Q, T),
                            _derived(dv.RelativeHumidity)),
      'ensemble_mean': ('ens_mean', (U,), _ensemble_mean),
      'spectrum_interpolation': ('spectrum_interp', (U,),
                                 _spectrum_interpolation),
      'bilinear_regrid': ('regrid_bilinear', (U,), _bilinear_regrid),
  }


FAMILIES = _families()


class WholeFakeContext(fake_ctx_column.ColumnFakeContext,
                       fake_ctx_dynamics.DynamicsFakeContext,
                       fake_ctx_thermo.ThermoFakeContext):
  """The stand-in with every entry `FAMILIES` calls."""


class KernelFailure(RuntimeError):
  pass


class FailingContext(WholeFakeContext):
  """A stand-in whose entries raise once the operands are uploaded and the
  output allocated."""
  failures = 0


def _fail(self, *args, **kwargs):
  del args, kwargs
  self.failures += 1
  raise KernelFailure('kernel failed')


for _entry in {entry for entry, _, _ in FAMILIES.values()}:
  setattr(FailingContext, _entry, _fail)


@pytest.mark.parametrize('family', FAMILIES)
def test_nothing_outlives_a_call(family):
  with fake_ctx.installed(WholeFakeContext) as fake:
    call = FAMILIES[family][2](2, _numpy)
    call()
    after_first = len(fake._bufs)  # pylint: disable=protected-access
    calls_first = len(fake.calls)
    call()
    assert len(fake._bufs) == after_first  # pylint: disable=protected-access
    assert len(fake.calls) == 2 * calls_first > 0


@pytest.mark.parametrize('family', FAMILIES)
def test_nothing_outlives_a_failed_entry(family):
  with fake_ctx.installed(FailingContext) as fake:
    call = FAMILIES[family][2](2, _numpy)
    with pytest.raises(KernelFailure):
      call()
    assert fake.failures == 1
    assert fake.h2d_bytes > 0  # the operands were uploaded
    assert not fake._bufs  # pylint: disable=protected-access


@pytest.mark.parametrize('family', FAMILIES)
def test_a_variable_without_cells_calls_no_entry(family):
  with fake_ctx.installed(WholeFakeContext) as fake:
    full = FAMILIES[family][2](2, _numpy)()
    fake.calls.clear()
    got = FAMILIES[family][2](0, _numpy)()
    assert fake.calls == []
    assert not fake._bufs  # pylint: disable=protected-access
  assert isinstance(got, np.ndarray)
  assert got.shape == (0,) + full.shape[1:] and got.dtype == full.dtype

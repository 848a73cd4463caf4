"""Derived variables on the hot path: `ZonalEnergySpectrum` with the API of
weatherbench2/derived_variables.py:29-56, 531-626.  The rFFT, the power
spectrum and the circumference scaling run in csrc/spectrum.cu.
The wind variables of derived_variables.py:59-338 -- wind speed, divergence,
vorticity, vertical velocity and the geostrophic / ageostrophic winds -- live in
_derived_wind.py (csrc/derived.cu, csrc/wind_dynamics.cu) and are re-exported
here.  The precipitation accumulations of derived_variables.py:471-528 and
685-720 live in _derived_precip.py (csrc/precip_accumulation.cu,
csrc/resample.cu) and are re-exported here.  The column integrals over
pressure level of derived_variables.py:212-228 and 365-430 -- eddy kinetic
energy, total column water and integrated water transport -- live in
_derived_column.py (csrc/column_integral.cu) and are re-exported here.  The
lapse rate and relative humidity of derived_variables.py:341-362 and 433-468
live in _derived_thermo.py (csrc/thermo.cu) and are re-exported here.
"""
from __future__ import annotations

import dataclasses
import typing as t

import numpy as np

from weatherbench2_b200 import _lib
from weatherbench2_b200 import _streamed
from weatherbench2_b200 import xarray_lite as xl

EARTH_RADIUS_M = 1000 * (6357 + 6378) / 2  # weatherbench2/schema.py:59


@dataclasses.dataclass
class DerivedVariable(xl.Boundary):
  """Derived variable base class (derived_variables.py:28-56)."""

  _boundary_methods = ('compute', 'compute_latitude_mean')

  @property
  def base_variables(self) -> list[str]:
    return []

  @property
  def core_dims(self):
    raise NotImplementedError

  @property
  def all_input_core_dims(self) -> set[str]:
    return set().union(*self.core_dims[0])

  def compute(self, dataset):
    raise NotImplementedError


@dataclasses.dataclass
class ZonalEnergySpectrum(DerivedVariable):
  """Energy spectrum along the zonal direction
  (derived_variables.py:531-626).

  S[0] = C |F[0]|^2, S[k] = 2 C |F[k]|^2 for k > 0 (the Nyquist bin included),
  F = rfft(f, norm='forward'), C = circumference of the latitude circle.
  Output dims: the input dims with `longitude` replaced by a trailing
  `zonal_wavenumber`; coords `frequency` (1 / m) and `wavelength` (m) with dims
  (zonal_wavenumber, latitude).
  """

  variable_name: str

  @property
  def base_variables(self) -> list[str]:
    return [self.variable_name]

  @property
  def core_dims(self):
    return (['longitude'],), ['zonal_wavenumber']

  def _circumference(self, latitude: np.ndarray) -> np.ndarray:
    """derived_variables.py:578-581."""
    circum_at_equator = 2 * np.pi * EARTH_RADIUS_M
    return np.cos(np.asarray(latitude) * np.pi / 180) * circum_at_equator

  def lon_spacing_m(self, dataset) -> xl.DataArray:
    """Spacing (meters) between longitudes (derived_variables.py:583-590)."""
    ds = xl.from_xarray(dataset)
    lon = ds['longitude'].values
    lat = ds['latitude'].values
    diffs = np.diff(lon)
    if np.max(np.abs(diffs - diffs[0])) > 1e-3:
      raise ValueError(f'Expected uniform longitude spacing. {lon=}')
    return xl.DataArray(self._circumference(lat) * diffs[0] / 360,
                        ('latitude',), {'latitude': lat})

  @staticmethod
  def _layout(da, sum_dim):
    """`da` as (outer..., latitude, longitude), `sum_dim` first so that field i
    adds to result slot i % nout; the result's outer dims and shape, nfield,
    the length of `sum_dim` (1 without it) and nout."""
    outer = tuple(d for d in da.dims if d not in ('latitude', 'longitude'))
    if sum_dim is not None:
      if sum_dim not in outer:
        raise ValueError(f'{sum_dim!r} is not a dimension of the data')
      outer = (sum_dim,) + tuple(d for d in outer if d != sum_dim)
    work = da.transpose(*(outer + ('latitude', 'longitude')))
    oshape = tuple(work.sizes[d] for d in outer)
    nfield = int(np.prod(oshape))  # 1 without outer dims
    nt = oshape[0] if sum_dim is not None else 1
    nout = nfield // nt
    if sum_dim is not None:
      outer, oshape = outer[1:], oshape[1:]
    return work, outer, oshape, nfield, nt, nout

  def compute(self, dataset, time_sum_dim: t.Optional[str] = None):
    """Zonal power at wavenumber and frequency (derived_variables.py:592-626).

    time_sum_dim (extension): when given, the spectrum is additionally summed
    over that dimension on the device (the script's `xbeam.Mean(['time'])`,
    scripts/compute_zonal_energy_spectrum.py:234, is sum / count); the
    dimension is dropped from the result.
    """
    spacing = self.lon_spacing_m(dataset).values
    da = dataset[self.variable_name]
    lat = dataset['latitude'].values
    lon = dataset['longitude'].values
    if 'latitude' not in da.dims or 'longitude' not in da.dims:
      raise ValueError(f'{self.variable_name} needs latitude and longitude')
    work, out_outer, oshape, nfield, _, nout = self._layout(da, time_sum_dim)
    ctx = _lib.default_context()
    nlat, nlon = lat.size, lon.size
    nk = nlon // 2 + 1
    scale = self._circumference(lat)
    summed = time_sum_dim is not None

    def device(x, _, out):
      if summed:  # the device entry adds into `out`
        out.zero_()
      ctx.zonal_spectrum(x.data_ptr(), nfield, nlat, nlon, scale,
                         out.data_ptr(), summed, nout)

    # host data is streamed through double-buffered staging; with a time sum
    # the accumulator stays in HBM and only the sum comes back
    values, = _streamed.place(
        work.data, [(oshape + (nlat, nk), np.float32)], device,
        lambda x, _, out: ctx.zonal_spectrum_host(
            x.ctypes.data, nfield, nlat, nlon, scale, out.ctypes.data, summed,
            nout), dtype=np.float32)
    dims = out_outer + ('latitude', 'zonal_wavenumber')
    base_frequency = np.fft.rfftfreq(nlon)  # derived_variables.py:614
    with np.errstate(divide='ignore'):
      frequency = base_frequency[:, None] / spacing[None, :]
      wavelength = 1 / frequency
    coords = {k: c for k, c in work.coords.items()
              if 'longitude' not in c.dims and all(d in dims for d in c.dims)}
    coords['zonal_wavenumber'] = xl.Coord(('zonal_wavenumber',), np.arange(nk))
    coords['frequency'] = xl.Coord(('zonal_wavenumber', 'latitude'), frequency,
                                   {'units': '1 / m'})
    coords['wavelength'] = xl.Coord(('zonal_wavenumber', 'latitude'),
                                    wavelength, {'units': 'm'})
    # the reference keeps the non-core dims in place and appends the new core
    # dim (apply_ufunc): (..., latitude, ..., zonal_wavenumber)
    ref_dims = tuple(d for d in da.dims if d != 'longitude' and
                     d != time_sum_dim) + ('zonal_wavenumber',)
    result = xl.DataArray(values, dims, coords, self.variable_name)
    if not xl._is_torch(work.data):  # pylint: disable=protected-access
      result = result.transpose(*ref_dims)
    return result


  def compute_latitude_mean(self, dataset, time_mean_dim: t.Optional[str] = None,
                            lat_slice: t.Optional[slice] = None):
    """North-star path (BASELINE.json): rFFT along longitude FOLLOWED BY the
    weighted meridional reduction, fused in one kernel
    (wb2_zonal_spectrum_latsum): the get_lat_weights-weighted latitude mean
    (weatherbench2/metrics.py:40-60) of `compute(dataset)`, optionally over the
    latitude band `lat_slice` (label-inclusive like SliceRegion) and averaged
    over `time_mean_dim`.  The per-latitude spectrum is never written (4 B read
    per cell, ~0 written).  Output dims: the remaining outer dims +
    `zonal_wavenumber`; no frequency / wavelength coordinates (they depend on
    latitude)."""
    from weatherbench2_b200 import _spatial as sp  # pylint: disable=import-outside-toplevel
    self.lon_spacing_m(dataset)  # uniform-longitude check (derived_variables.py:583-590)
    da = dataset[self.variable_name]
    lat = dataset['latitude'].values
    lon = dataset['longitude'].values
    work, out_outer, oshape, nfield, nt, nout = self._layout(da,
                                                             time_mean_dim)
    nlat, nlon = lat.size, lon.size
    nk = nlon // 2 + 1
    w = sp.lat_weights(lat)
    if lat_slice is not None:
      lo = -np.inf if lat_slice.start is None else lat_slice.start
      hi = np.inf if lat_slice.stop is None else lat_slice.stop
      w = w * ((lat >= lo) & (lat <= hi))
    if not w.sum() > 0:
      raise ValueError('the latitude band selects no latitude')
    scale = self._circumference(lat) * w / w.sum() / nt
    ctx = _lib.default_context()
    values, = _streamed.place(
        work.data, [(oshape + (nk,), np.float32)],
        lambda x, _, out: ctx.zonal_spectrum_latsum(
            x.data_ptr(), nfield, nlat, nlon, scale, out.data_ptr(), nout),
        lambda x, _, out: ctx.zonal_spectrum_latsum_host(
            x.ctypes.data, nfield, nlat, nlon, scale, out.ctypes.data, nout),
        dtype=np.float32)
    dims = out_outer + ('zonal_wavenumber',)
    coords = {k: c for k, c in work.coords.items()
              if all(d in out_outer for d in c.dims)}
    coords['zonal_wavenumber'] = xl.Coord(('zonal_wavenumber',), np.arange(nk))
    return xl.DataArray(values, dims, coords, self.variable_name)


@xl.boundary
def interpolate_spectral_frequencies(spectrum, wavenumber_dim: str,
                                     frequencies=None, method: str = 'linear'):
  """Interpolate the frequencies of `spectrum` (as produced by
  ZonalEnergySpectrum.compute) to common values
  (weatherbench2/derived_variables.py:629-682): every latitude row lives on its
  own frequency axis; the result replaces `wavenumber_dim` by `frequency`, NaN
  where a common frequency lies outside a row's range.  Default frequencies:
  the narrowest range present, `spectrum.sizes[wavenumber_dim]` points
  (:658-664).  Linear interpolation only (the kernel is a gather + lerp)."""
  if method != 'linear':
    raise NotImplementedError('only method="linear" runs on the device')
  freq = spectrum.coords['frequency']
  if set(freq.dims) != {wavenumber_dim, 'latitude'}:
    raise ValueError(f'{freq.dims=} was not a permutation of '
                     f'("{wavenumber_dim}", "latitude")')
  fv = np.asarray(freq.values, dtype=np.float64)
  if freq.dims[0] != wavenumber_dim:
    fv = fv.T  # (wavenumber, latitude)
  nk, nlat = fv.shape
  if frequencies is None:
    freq_min = fv.max(axis=1).min()
    freq_max = fv.min(axis=1).max()
    frequencies = np.linspace(freq_min, freq_max, num=nk)
  frequencies = np.asarray(frequencies, dtype=np.float64)
  if frequencies.ndim != 1:
    raise ValueError(f'Expected 1-D frequencies, found {frequencies.shape=}')
  table = np.ascontiguousarray(fv.T)  # (latitude, wavenumber), increasing in k
  if nk < 2 or not (np.diff(table, axis=1) > 0).all():
    raise ValueError('the frequency coordinate must increase with wavenumber')
  outer = tuple(d for d in spectrum.dims
                if d not in ('latitude', wavenumber_dim))
  work = spectrum.transpose(*(outer + ('latitude', wavenumber_dim)))
  data = work.data
  oshape = tuple(work.sizes[d] for d in outer)
  nfield = int(np.prod(oshape)) if oshape else 1
  nf = frequencies.size
  ctx = _lib.default_context()
  values, = _streamed.run_whole(
      [data], [(oshape + (nlat, nf), np.float32)],
      lambda i, o: ctx.spectrum_interp(i[0], nfield, nlat, nk, table,
                                       frequencies, o[0]),
      dtype=np.float32)
  dims = outer + ('latitude', 'frequency')
  coords = {k: c for k, c in work.coords.items()
            if wavenumber_dim not in c.dims and k not in ('frequency',
                                                           'wavelength')}
  coords['frequency'] = xl.Coord(('frequency',), frequencies)
  with np.errstate(divide='ignore'):
    # "Interp didn't deal well with the infinite wavelength, so just reset"
    coords['wavelength'] = xl.Coord(('frequency',), 1 / frequencies,
                                    {'units': 'm'})
  result = xl.DataArray(values, dims, coords, spectrum.name, spectrum.attrs)
  # the reference's groupby('latitude').apply keeps latitude where it was and
  # puts frequency in the wavenumber's place
  ref_dims = tuple('frequency' if d == wavenumber_dim else d
                   for d in spectrum.dims)
  if not xl._is_torch(values):  # pylint: disable=protected-access
    result = result.transpose(*ref_dims)
  return result


# Wind variables live in _derived_wind.py (they need DerivedVariable).
from weatherbench2_b200._derived_wind import (  # noqa: E402  pylint: disable=wrong-import-position
    AgeostrophicWindSpeed, GeostrophicWindSpeed, UComponentOfAgeostrophicWind,
    UComponentOfGeostrophicWind, VComponentOfAgeostrophicWind,
    VComponentOfGeostrophicWind, VerticalVelocity, WindDivergence,
    WindSpeed, WindVorticity, _3DWindVariable, _AgeostrophicWindVariable,
    _GeostrophicWindVariable)
from weatherbench2_b200._derived_precip import (  # noqa: E402  pylint: disable=wrong-import-position
    AggregatePrecipitationAccumulation, PrecipitationAccumulation)
from weatherbench2_b200._derived_column import (  # noqa: E402  pylint: disable=wrong-import-position
    EddyKineticEnergy, IntegratedWaterTransport, TotalColumnWater)
from weatherbench2_b200._derived_thermo import (  # noqa: E402  pylint: disable=wrong-import-position
    LapseRate, RelativeHumidity)

# The named derived variables of weatherbench2/derived_variables.py:724-773 that
# have a device implementation: wind speed, the horizontal-derivative family
# (divergence, vorticity, vertical velocity, geostrophic and ageostrophic
# winds), the column integrals (eddy kinetic energy, total column water,
# integrated vapor transport) and the precipitation accumulations.  The
# reference's 'lapse_rate' and 'relative_humidity' entries are not registered
# yet: their classes, LapseRate and RelativeHumidity, run on the device and
# work anywhere a DerivedVariable is accepted, but asking this table for either
# name raises KeyError until a follow-up adds the two entries.
DERIVED_VARIABLE_DICT = {
    'wind_speed': WindSpeed(u_name='u_component_of_wind',
                            v_name='v_component_of_wind'),
    '10m_wind_speed': WindSpeed(u_name='10m_u_component_of_wind',
                                v_name='10m_v_component_of_wind'),
    'divergence': WindDivergence(),
    'vorticity': WindVorticity(),
    'vertical_velocity': VerticalVelocity(),
    'eddy_kinetic_energy': EddyKineticEnergy(),
    'geostrophic_wind_speed': GeostrophicWindSpeed(),
    'u_component_of_geostrophic_wind': UComponentOfGeostrophicWind(),
    'v_component_of_geostrophic_wind': VComponentOfGeostrophicWind(),
    'ageostrophic_wind_speed': AgeostrophicWindSpeed(),
    'u_component_of_ageostrophic_wind': UComponentOfAgeostrophicWind(),
    'v_component_of_ageostrophic_wind': VComponentOfAgeostrophicWind(),
    'total_column_vapor': TotalColumnWater(
        water_species_name='specific_humidity'
    ),
    'total_column_liquid': TotalColumnWater(
        water_species_name='specific_cloud_liquid_water_content'
    ),
    'total_column_ice': TotalColumnWater(
        water_species_name='specific_cloud_ice_water_content'
    ),
    'integrated_vapor_transport': IntegratedWaterTransport(),
    'total_precipitation_6hr': PrecipitationAccumulation(
        total_precipitation_name='total_precipitation',
        accumulation_hours=6,
        lead_time_name='prediction_timedelta',
    ),
    'total_precipitation_24hr': PrecipitationAccumulation(
        total_precipitation_name='total_precipitation',
        accumulation_hours=24,
        lead_time_name='prediction_timedelta',
    ),
    'total_precipitation_24hr_from_6hr': AggregatePrecipitationAccumulation(
        accumulation_hours=24,
        lead_time_name='prediction_timedelta',
    ),
    'total_precipitation_24hr_from_12hr': AggregatePrecipitationAccumulation(
        accumulation_hours=24,
        lead_time_name='prediction_timedelta',
        raw_accumulation_name='total_precipitation_12hr',
        raw_accumulation_hours=12,
    ),
}

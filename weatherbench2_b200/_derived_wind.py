"""Wind derived variables -- same classes as
weatherbench2/derived_variables.py:59-99 and 132-338 -- computed on the device
(csrc/derived.cu, csrc/wind_dynamics.cu).  Imported into
`weatherbench2_b200.derived_variables`.
"""
from __future__ import annotations

import dataclasses
import math

import numpy as np

from weatherbench2_b200 import _lib
from weatherbench2_b200 import _streamed
from weatherbench2_b200 import derived_variables as dv
from weatherbench2_b200 import xarray_lite as xl


@dataclasses.dataclass
class _WindVariable(dv.DerivedVariable):
  """A variable derived from the U and V wind components
  (derived_variables.py:59-74)."""

  u_name: str
  v_name: str

  @property
  def base_variables(self) -> list[str]:
    return [self.u_name, self.v_name]


@dataclasses.dataclass
class WindSpeed(_WindVariable):
  """Wind speed sqrt(u**2 + v**2) (derived_variables.py:77-99).  NumPy in ->
  NumPy out; a CUDA tensor in -> a CUDA tensor that the metric kernels read in
  place."""

  @property
  def core_dims(self):
    return ([], []), []

  def compute(self, dataset):
    u, v = dataset[self.u_name], dataset[self.v_name]
    if u.dims != v.dims or u.shape != v.shape:
      v = v.transpose(*u.dims)
      if u.shape != v.shape:
        raise ValueError(f'{self.u_name} and {self.v_name} differ in shape')
    ctx = _lib.default_context()
    n = math.prod(u.shape)
    data, = _streamed.run_whole(
        [u.data, v.data], [(u.shape, np.float32)],
        lambda i, o: ctx.wind_speed(i[0], i[1], o[0], n), dtype=np.float32)
    coords = {k: c for k, c in u.coords.items()}
    return xl.DataArray(data, u.dims, coords)


# ---- horizontal derivatives (derived_variables.py:102-338) -------------------
# `kind` of wb2_wind_dynamics (include/wb2b200.h)
DIVERGENCE, VORTICITY, VERTICAL_VELOCITY = 0, 1, 2
GEOSTROPHIC_WIND_SPEED, U_GEOSTROPHIC, V_GEOSTROPHIC = 3, 4, 5
AGEOSTROPHIC_WIND_SPEED, U_AGEOSTROPHIC, V_AGEOSTROPHIC = 6, 7, 8

OMEGA = 7.292e-5  # radians / second (derived_variables.py:234)


def check_same_grid(names, das):
  """ValueError unless every variable of `das` (named `names`) has the first
  one's dims, in any order, and sizes."""
  for name, da in zip(names[1:], das[1:]):
    if set(da.dims) != set(das[0].dims) or any(
        da.sizes[d] != das[0].sizes[d] for d in das[0].dims):
      raise ValueError(f'{names[0]!r} and {name!r} differ in dims or shape')


def gradient_table(coord) -> tuple[np.ndarray, bool]:
  """np.gradient's coefficients (edge_order=1) along one axis with coordinate
  `coord`, as the [n][3] float64 table wb2_wind_dynamics reads, and whether
  the spacing is uniform (every diff equal to the first, np.gradient's test).
  The expressions are np.gradient's, so the coefficients are bit-identical."""
  x = np.asarray(coord, dtype=np.float64)
  if x.ndim != 1 or x.size < 2:
    raise ValueError('Shape of array too small to calculate a numerical '
                     'gradient, at least (edge_order + 1) elements are required.')
  dx = np.diff(x)
  uniform = bool((dx == dx[0]).all())
  table = np.zeros((x.size, 3))
  if uniform:
    table[:, 0] = 2. * dx[0]
    table[0, 0] = table[-1, 0] = dx[0]
  else:
    dx1, dx2 = dx[0:-1], dx[1:]
    table[1:-1, 0] = -(dx2) / (dx1 * (dx1 + dx2))
    table[1:-1, 1] = (dx2 - dx1) / (dx1 * dx2)
    table[1:-1, 2] = dx1 / (dx2 * (dx1 + dx2))
    table[0, 0], table[-1, 0] = dx[0], dx[-1]
  return table, uniform


def coriolis_parameter(latitude) -> np.ndarray:
  """2 * omega * sin(deg2rad(lat)) (derived_variables.py:234-237)."""
  return 2 * OMEGA * np.sin(np.deg2rad(np.asarray(latitude, np.float64)))


def wind_dynamics(dataset, kind: int, u_name=None, v_name=None, z_name=None):
  """One wb2_wind_dynamics call on the named variables of `dataset`.  The
  result keeps the first input's dims and coords; float32, on the device when
  an input is a CUDA tensor, else NumPy.  Float64 data is cast to float32 and
  float32 coordinates are taken as float64 (DESIGN.md, "Wind dynamics")."""
  names = [n for n in (u_name, v_name, z_name) if n is not None]
  das = [dataset[n] for n in names]  # KeyError for a missing base variable
  ref = das[0]
  for d in ('latitude', 'longitude'):
    if d not in ref.dims or d not in ref.coords:
      raise ValueError(f'{ref.name} needs a {d!r} dimension and coordinate')
  vertical = kind == VERTICAL_VELOCITY
  if vertical:
    if 'level' not in ref.coords:
      raise KeyError('level')
    if 'level' not in ref.dims:
      raise ValueError(f'{ref.name} has no "level" dimension')
  spatial = (('latitude', 'longitude')
             if ref.dims.index('latitude') < ref.dims.index('longitude')
             else ('longitude', 'latitude'))
  lead = (('level',) if vertical else ())
  outer = tuple(d for d in ref.dims if d not in spatial + lead)
  work = outer + lead + spatial
  check_same_grid(names, das)
  lat = ref.coords['latitude'].values
  lon = ref.coords['longitude'].values
  lat_tab, lat_uniform = gradient_table(lat)
  lon_tab, lon_uniform = gradient_table(lon)
  cos_lat = np.cos(np.deg2rad(np.asarray(lat, np.float64)))
  coriolis = (coriolis_parameter(lat) if kind >= GEOSTROPHIC_WIND_SPEED
              else None)
  pressure = (100 * np.asarray(ref.coords['level'].values, np.float64)
              if vertical else None)
  nlat, nlon = lat.size, lon.size
  nlev = ref.sizes['level'] if vertical else 1
  shape = tuple(ref.sizes[d] for d in work)
  nouter = int(np.prod(shape[:len(outer)])) if outer else 1
  strides = (nlon, 1) if spatial[0] == 'latitude' else (1, nlat)
  ctx = _lib.default_context()

  def call(ptrs, out):
    by_name = dict(zip(names, ptrs))
    ctx.wind_dynamics(kind, by_name.get(u_name), by_name.get(v_name),
                      by_name.get(z_name), nouter, nlev, nlat, nlon, *strides,
                      lat_tab, lat_uniform, lon_tab, lon_uniform, cos_lat,
                      coriolis, pressure, out[0])

  data, = _streamed.run_whole([da.transpose(*work).data for da in das],
                              [(shape, np.float32)], call, dtype=np.float32)
  coords = {k: c for k, c in ref.coords.items()}
  result = xl.DataArray(data, work, coords).transpose(*ref.dims)
  if xl._is_torch(result.data):  # pylint: disable=protected-access
    result = xl.DataArray(result.data.contiguous(), result.dims, coords)
  return result


@dataclasses.dataclass
class _3DWindVariable(dv.DerivedVariable):
  """A variable derived from 3D U and V wind components
  (derived_variables.py:132-146)."""

  u_name: str = 'u_component_of_wind'
  v_name: str = 'v_component_of_wind'

  @property
  def base_variables(self) -> list[str]:
    return [self.u_name, self.v_name]


@dataclasses.dataclass
class WindDivergence(_3DWindVariable):
  """Horizontal wind divergence _d_dx(u) + _d_dy(v), 1 / s
  (derived_variables.py:149-161)."""

  @property
  def core_dims(self):
    lon_lat = ['longitude', 'latitude']
    return (lon_lat, lon_lat), lon_lat

  def compute(self, dataset):
    return wind_dynamics(dataset, DIVERGENCE, self.u_name, self.v_name)


@dataclasses.dataclass
class WindVorticity(_3DWindVariable):
  """Relative vorticity _d_dx(v) - _d_dy(u), 1 / s, without the spherical
  metric term, as in the reference (derived_variables.py:164-176)."""

  @property
  def core_dims(self):
    lon_lat = ['longitude', 'latitude']
    return (lon_lat, lon_lat), lon_lat

  def compute(self, dataset):
    return wind_dynamics(dataset, VORTICITY, self.u_name, self.v_name)


@dataclasses.dataclass
class VerticalVelocity(_3DWindVariable):
  """Pressure vertical velocity omega = -integral of the divergence over
  pressure (Pa / s), hydrostatic: scipy's cumulative_trapezoid along `level`
  with x = 100 * level and initial 0 (derived_variables.py:179-209).  Needs a
  `level` dimension and coordinate (hPa)."""

  @property
  def core_dims(self):
    zxy = ['level', 'longitude', 'latitude']
    return (zxy, zxy), zxy

  def compute(self, dataset):
    return wind_dynamics(dataset, VERTICAL_VELOCITY, self.u_name, self.v_name)


@dataclasses.dataclass
class _GeostrophicWindVariable(dv.DerivedVariable):
  """Base class of the geostrophic winds -_d_dy(z) / f, _d_dx(z) / f
  (derived_variables.py:231-260).  They are +-inf or NaN on the equator, where
  f = 0; the reference leaves the choice of region to the user."""

  geopotential_name: str = 'geopotential'

  @property
  def base_variables(self) -> list[str]:
    return [self.geopotential_name]

  @property
  def core_dims(self):
    lon_lat = ['longitude', 'latitude']
    return (lon_lat,), lon_lat


@dataclasses.dataclass
class GeostrophicWindSpeed(_GeostrophicWindVariable):
  """Geostrophic wind speed (derived_variables.py:263-276), a balance
  diagnostic for AI weather models (https://arxiv.org/abs/2309.08473)."""

  def compute(self, dataset):
    return wind_dynamics(dataset, GEOSTROPHIC_WIND_SPEED,
                         z_name=self.geopotential_name)


class UComponentOfGeostrophicWind(_GeostrophicWindVariable):
  """East-west component of geostrophic wind (derived_variables.py:279-284)."""

  def compute(self, dataset):
    return wind_dynamics(dataset, U_GEOSTROPHIC, z_name=self.geopotential_name)


class VComponentOfGeostrophicWind(_GeostrophicWindVariable):
  """North-south component of geostrophic wind
  (derived_variables.py:287-292)."""

  def compute(self, dataset):
    return wind_dynamics(dataset, V_GEOSTROPHIC, z_name=self.geopotential_name)


@dataclasses.dataclass
class _AgeostrophicWindVariable(dv.DerivedVariable):
  """Base class of the ageostrophic winds u - u_geo, v - v_geo
  (derived_variables.py:295-310)."""

  u_name: str = 'u_component_of_wind'
  v_name: str = 'v_component_of_wind'
  geopotential_name: str = 'geopotential'

  @property
  def base_variables(self) -> list[str]:
    return [self.u_name, self.v_name, self.geopotential_name]

  @property
  def core_dims(self):
    lon_lat = ['longitude', 'latitude']
    return (lon_lat, lon_lat, lon_lat), lon_lat


class AgeostrophicWindSpeed(_AgeostrophicWindVariable):
  """Ageostrophic wind speed (derived_variables.py:313-320)."""

  def compute(self, dataset):
    return wind_dynamics(dataset, AGEOSTROPHIC_WIND_SPEED, self.u_name,
                         self.v_name, self.geopotential_name)


class UComponentOfAgeostrophicWind(_AgeostrophicWindVariable):
  """East-west component of ageostrophic wind (derived_variables.py:323-329)."""

  def compute(self, dataset):
    return wind_dynamics(dataset, U_AGEOSTROPHIC, self.u_name,
                         z_name=self.geopotential_name)


class VComponentOfAgeostrophicWind(_AgeostrophicWindVariable):
  """North-south component of ageostrophic wind
  (derived_variables.py:332-338)."""

  def compute(self, dataset):
    return wind_dynamics(dataset, V_AGEOSTROPHIC, v_name=self.v_name,
                         z_name=self.geopotential_name)

"""TEST ORACLE: the horizontal-derivative derived variables of
weatherbench2/derived_variables.py:102-338 restated in NumPy, step for step as
the reference computes them on float32 data with float64 coordinates:
np.gradient(edge_order=1) stored as float32 (xarray's `differentiate`), `_d_dx`
in float64 with the poles zeroed, `_d_dy` as a float32 division by the Python
float M, the combinations in float64, and scipy's cumulative_trapezoid along
`level`.  Results are float64; the kernels round them once to float32.  It does
not import the product."""
import numpy as np
import scipy.integrate

EARTH_RADIUS_M = 1000 * (6357 + 6378) / 2  # weatherbench2/schema.py:59
METERS_PER_DEGREE = 2 * np.pi * EARTH_RADIUS_M / 360
OMEGA = 7.292e-5

KINDS = ('divergence', 'vorticity', 'vertical_velocity',
         'geostrophic_wind_speed', 'u_component_of_geostrophic_wind',
         'v_component_of_geostrophic_wind', 'ageostrophic_wind_speed',
         'u_component_of_ageostrophic_wind', 'v_component_of_ageostrophic_wind')


def _along(values, dims, dim):
  """1-D coordinate `values` shaped to broadcast along `dim` of `dims`."""
  shape = [1] * len(dims)
  shape[dims.index(dim)] = -1
  return np.asarray(values, np.float64).reshape(shape)


def gradient(f, coord, axis):
  """xarray's differentiate: np.gradient on float64 coordinates, edge_order=1,
  result in f's dtype."""
  return np.gradient(f, np.asarray(coord, np.float64), edge_order=1, axis=axis)


def d_dx(f, dims, lat, lon):
  """derived_variables.py:110-117: float64."""
  cos = np.cos(np.deg2rad(_along(lat, dims, 'latitude')))
  with np.errstate(divide='ignore', invalid='ignore'):
    g = gradient(f, lon, dims.index('longitude')) / cos / METERS_PER_DEGREE
  return np.where(cos > 1e-6, g, 0.0)


def d_dy(f, dims, lat):
  """derived_variables.py:120-121: the Python float is weak, so float32 data
  stays float32."""
  return gradient(f, lat, dims.index('latitude')) / METERS_PER_DEGREE


def geostrophic(z, dims, lat, lon):
  """derived_variables.py:231-244: (u_geo, v_geo), float64."""
  f = 2 * OMEGA * np.sin(np.deg2rad(_along(lat, dims, 'latitude')))
  with np.errstate(divide='ignore', invalid='ignore'):
    return -d_dy(z, dims, lat) / f, d_dx(z, dims, lat, lon) / f


def compute(kind, dims, lat, lon, u=None, v=None, z=None, level=None):
  """The reference's compute() of derived variable `kind` (a name of KINDS) on
  arrays with dimension names `dims`; float64 result in the same layout."""
  dims = tuple(dims)
  with np.errstate(invalid='ignore', over='ignore'):
    if kind == 'divergence':
      return d_dx(u, dims, lat, lon) + d_dy(v, dims, lat)
    if kind == 'vorticity':
      return d_dx(v, dims, lat, lon) - d_dy(u, dims, lat)
    if kind == 'vertical_velocity':
      div = d_dx(u, dims, lat, lon) + d_dy(v, dims, lat)
      pressure = 100 * np.asarray(level, np.float64)
      return scipy.integrate.cumulative_trapezoid(
          -div, x=pressure, axis=dims.index('level'), initial=0)
    ug, vg = geostrophic(z, dims, lat, lon)
    if kind == 'geostrophic_wind_speed':
      return np.sqrt(ug**2 + vg**2)
    if kind == 'u_component_of_geostrophic_wind':
      return ug
    if kind == 'v_component_of_geostrophic_wind':
      return vg
    if kind == 'ageostrophic_wind_speed':
      return np.sqrt((u - ug)**2 + (v - vg)**2)
    if kind == 'u_component_of_ageostrophic_wind':
      return u - ug
    if kind == 'v_component_of_ageostrophic_wind':
      return v - vg
  raise ValueError(kind)


def inputs_of(kind):
  """Which of u, v, z the reference reads for `kind`."""
  if 'ageostrophic' in kind:
    return {'ageostrophic_wind_speed': 'uvz',
            'u_component_of_ageostrophic_wind': 'uz',
            'v_component_of_ageostrophic_wind': 'vz'}[kind]
  return 'z' if 'geostrophic' in kind else 'uv'

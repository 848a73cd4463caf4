"""TEST INFRASTRUCTURE: seeded wind / geopotential datasets for the wind
dynamics tests (tests/test_wind_dynamics_cpu.py, tests/test_wind_dynamics_gpu.py)."""
import numpy as np

NAMES = {'u': 'u_component_of_wind', 'v': 'v_component_of_wind',
         'z': 'geopotential'}


def grid(name):
  """(latitude, longitude) of a named test grid."""
  if name == 'uniform721':  # 0.25 degrees, poles and equator included
    return np.linspace(-90, 90, 721), np.arange(1440) * 0.25
  if name == 'nonuniform32':  # 32 rows, poles and an exact equator
    return np.sort(np.r_[np.linspace(-90, 90, 31), 3.0]), np.linspace(0, 355, 64)
  if name == 'descending':
    return np.linspace(90, -90, 19), np.arange(36) * 10.0
  if name == 'regional':  # no poles, no equator, non-uniform longitude
    return np.linspace(25, 65, 17), np.cumsum(np.r_[-30, np.full(24, 2.5)] +
                                              np.r_[0, np.tile([0, .5], 12)])
  raise ValueError(name)


def fields(shape, seed, nan=True):
  """u, v (m/s) and z (m^2/s^2) float32 with a few NaN cells."""
  rs = np.random.RandomState(seed)
  u = rs.normal(scale=10, size=shape).astype(np.float32)
  v = rs.normal(scale=10, size=shape).astype(np.float32)
  z = (5e4 + rs.normal(scale=300, size=shape)).astype(np.float32)
  if nan:
    for x, k in ((u, 7), (v, 3 * shape[-1] + 1), (z, 2 * shape[-1] + 5)):
      x.reshape(-1)[k] = np.nan
  return {'u': u, 'v': v, 'z': z}


def dataset(xl, dims, lat, lon, data, level=(1000, 850, 500), ntime=2,
            wrap=None):
  """xarray_lite Dataset of the three variables with dimension order `dims`
  (a permutation of some of time, level, latitude, longitude).  `wrap` maps
  each array before it goes in (e.g. to a CUDA tensor)."""
  coords = {'time': np.arange(ntime), 'level': np.asarray(level),
            'latitude': lat, 'longitude': lon}
  coords = {k: c for k, c in coords.items() if k in dims}
  wrap = wrap or (lambda a: a)
  return xl.Dataset({NAMES[k]: (dims, wrap(a)) for k, a in data.items()},
                    coords)


def shape_of(dims, lat, lon, level=(1000, 850, 500), ntime=2):
  sizes = {'time': ntime, 'level': len(level), 'latitude': lat.size,
           'longitude': lon.size}
  return tuple(sizes[d] for d in dims)

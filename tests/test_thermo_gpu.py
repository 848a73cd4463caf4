"""GPU: wb2_lapse_rate and wb2_relative_humidity against tests/thermo_oracle.py
at 721 x 1440 with 13 and 37 levels, in both spatial layouts and with the
level axis innermost, in float32 and float64, with NaN cells and a dz == 0
column; an exhaustive sweep of every float32 temperature in [180, 330] K; and
the reference's own vectors."""
import os

import numpy as np
import pytest

import thermo_oracle as to

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')
if not torch.cuda.is_available():
  pytest.skip('needs a CUDA device', allow_module_level=True)

HERE = os.path.dirname(os.path.abspath(__file__))
T, Z, Q = 'temperature', 'geopotential', 'specific_humidity'
WB2_13 = np.array([50, 100, 150, 200, 250, 300, 400, 500, 600, 700, 850, 925,
                   1000])
ERA5_37 = np.array([1, 2, 3, 5, 7, 10, 20, 30, 50, 70, 100, 125, 150, 175, 200,
                    225, 250, 300, 350, 400, 450, 500, 550, 600, 650, 700, 750,
                    775, 800, 825, 850, 875, 900, 925, 950, 975, 1000])
LAT, LON = np.linspace(-90, 90, 721), np.arange(1440) * 0.25
LAYOUTS = {'lat_lon': ('level', 'latitude', 'longitude'),
           'lon_lat': ('level', 'longitude', 'latitude'),
           'level_innermost': ('latitude', 'longitude', 'level')}


def _height(level):
  return 44330.8 * (1 - (np.asarray(level, np.float64) / 1013.25) ** 0.190263)


def _fields(dims, level, dtype, seed=0):
  """Realistic profiles with NaN cells and one column of constant
  geopotential (dz == 0)."""
  sizes = {'level': level.size, 'latitude': LAT.size, 'longitude': LON.size}
  shape = tuple(sizes[d] for d in dims)
  rs = np.random.default_rng(seed)
  prof = [None] * len(dims)
  prof[dims.index('level')] = slice(None)
  h = _height(level)[tuple(prof)]
  f = {T: (288.15 - 6.5e-3 * np.minimum(h, 11000) +
           rs.standard_normal(size=shape, dtype=np.float32) * 5).astype(dtype),
       Z: (9.81 * h + rs.standard_normal(size=shape, dtype=np.float32) * 50
           ).astype(dtype),
       Q: (np.abs(rs.standard_normal(size=shape, dtype=np.float32)) * 6e-3 *
           np.exp(-h / 2500)).astype(dtype)}
  for k, n in ((T, 3), (Z, 5), (Q, 7)):
    f[k].reshape(-1)[rs.integers(0, f[k].size, n)] = np.nan
  col = [300] * len(dims)
  col[dims.index('level')] = slice(None)
  f[Z][tuple(col)] = f[Z][tuple(col)][0]
  return f


def _dataset(fields, dims, level, device=True):
  from weatherbench2_b200 import xarray_lite as xl
  coords = {'level': level, 'latitude': LAT, 'longitude': LON}
  return xl.Dataset(
      {k: (dims, torch.from_numpy(a).cuda() if device else a)
       for k, a in fields.items()}, coords)


def _pressure(level, dims):
  shape = [1] * len(dims)
  shape[dims.index('level')] = -1
  return np.asarray(level).reshape(shape)


def _assert_rh(got, t, q, p):
  """Bit-equal to the oracle, except where the float64 exp lies within one
  float64 ulp of a float32 rounding boundary: there either float32 neighbour
  of the rounded exp is accepted (float32 data); float64 data is held to the
  header's bound."""
  dtype = to.data_dtype(t, q)
  want, svp = to.relative_humidity(t, q, p, with_svp=True)
  assert got.dtype == want.dtype
  if dtype == np.float64:
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
    ok = np.isnan(want) | (np.abs(got - want) <= to.rh_bound(want, svp, p,
                                                            dtype))
    assert ok.all()
    return 0
  x = to.bolton_argument(t)
  flagged, other = to.exp_boundary(x)
  same = (got == want) | (np.isnan(got) & np.isnan(want))
  alt = to.relative_humidity(t, q, p, e=other)
  same_alt = (got == alt) | (np.isnan(got) & np.isnan(alt))
  assert (same | (flagged & same_alt)).all(), (
      int((~same).sum()), int((~same & ~flagged).sum()))
  return int((~same).sum())


@pytest.mark.parametrize('nlev', [13, 37])
@pytest.mark.parametrize('layout', list(LAYOUTS))
@pytest.mark.parametrize('dtype', [np.float32, np.float64])
def test_lapse_rate_is_bit_equal_to_the_oracle(nlev, layout, dtype):
  from weatherbench2_b200 import derived_variables as dv
  dims = LAYOUTS[layout]
  level = WB2_13 if nlev == 13 else ERA5_37
  f = _fields(dims, level, dtype, seed=nlev)
  got = dv.LapseRate().compute(_dataset({T: f[T], Z: f[Z]}, dims, level))
  assert got.dims == dims and got.data.is_cuda
  out = got.data.cpu().numpy()
  assert out.dtype == dtype
  want = to.lapse_rate(f[T], f[Z], level, dims.index('level'))
  np.testing.assert_array_equal(out, want)
  assert np.isinf(want).any() and np.isnan(want).any()


@pytest.mark.parametrize('nlev', [13, 37])
@pytest.mark.parametrize('layout', list(LAYOUTS))
@pytest.mark.parametrize('dtype,level_dtype', [
    (np.float32, np.int64), (np.float32, np.float32), (np.float64, np.int64)])
def test_relative_humidity_matches_the_oracle(nlev, layout, dtype, level_dtype):
  from weatherbench2_b200 import derived_variables as dv
  dims = LAYOUTS[layout]
  level = (WB2_13 if nlev == 13 else ERA5_37).astype(level_dtype)
  f = _fields(dims, level, dtype, seed=nlev + 1)
  got = dv.RelativeHumidity().compute(_dataset({T: f[T], Q: f[Q]}, dims,
                                               level))
  assert got.dims == dims and got.data.is_cuda
  n = _assert_rh(got.data.cpu().numpy(), f[T], f[Q], _pressure(level, dims))
  print(f'{layout} {nlev} {np.dtype(dtype).name} levels '
        f'{np.dtype(level_dtype).name}: {n} boundary cells differ')


def test_every_float32_temperature_against_numpy():
  """Every float32 temperature in [180, 330] K at four pressures, against
  NumPy's own arithmetic of the reference's expression, within the header's
  bound; and against the oracle as in _assert_rh."""
  from weatherbench2_b200 import derived_variables as dv, xarray_lite as xl
  t = np.arange(np.float32(180).view(np.int32),
                np.float32(330).view(np.int32) + 1,
                dtype=np.int32).view(np.float32)
  assert t.size == 7405569
  level = np.array([50, 300, 700, 1000])
  tt = np.broadcast_to(t, (level.size, t.size)).copy()
  rs = np.random.default_rng(9)
  qq = (np.abs(rs.standard_normal(size=tt.shape, dtype=np.float32)) * 5e-3
        ).astype(np.float32)
  ds = xl.Dataset({T: (('level', 'cell'), tt), Q: (('level', 'cell'), qq)},
                  {'level': level})
  got = dv.RelativeHumidity().compute(ds)
  assert isinstance(got.data, np.ndarray) and got.data.dtype == np.float64
  p = level[:, None]
  with np.errstate(all='ignore'):
    vapour = 6.112 * np.exp(17.67 * (tt - 273.15) / (tt - 29.65))
    numpy_rh = (qq / (1 - qq)) / (0.622 * vapour / (p - vapour))
  _, svp = to.relative_humidity(tt, qq, p, with_svp=True)
  bound = to.rh_bound(numpy_rh, svp, p, np.float32)
  gap = np.abs(got.values - numpy_rh)
  np.testing.assert_array_equal(np.isnan(got.values), np.isnan(numpy_rh))
  assert (np.isnan(numpy_rh) | (gap <= bound)).all()
  finite = np.isfinite(numpy_rh) & (numpy_rh != 0)
  print('largest gap / bound', float(np.max(gap[finite] / bound[finite])))
  _assert_rh(got.values, tt, qq, p)


def test_device_and_host_operands():
  from weatherbench2_b200 import derived_variables as dv
  dims = ('level', 'latitude', 'longitude')
  level = np.array([500, 850])
  f = {k: a[:, :40, :64].copy() for k, a in _fields(
      ('level', 'latitude', 'longitude'), level, np.float32).items()}

  def small(device):
    from weatherbench2_b200 import xarray_lite as xl
    return xl.Dataset({k: (dims, torch.from_numpy(a).cuda() if device else a)
                       for k, a in f.items()},
                      {'level': level, 'latitude': LAT[:40],
                       'longitude': LON[:64]})

  for var in (dv.LapseRate(), dv.RelativeHumidity()):
    on_device = var.compute(small(True))
    on_host = var.compute(small(False))
    assert on_device.data.is_cuda and isinstance(on_host.data, np.ndarray)
    np.testing.assert_array_equal(on_device.data.cpu().numpy(), on_host.data)


def test_reference_vectors():
  from weatherbench2_b200 import derived_variables as dv, xarray_lite as xl
  vec = np.load(os.path.join(HERE, 'golden', 'reference_thermo_vectors.npz'))
  names = sorted({k.split('|')[0] for k in vec.files} - {'metpy'})
  for name in names:
    g = lambda k: vec[f'{name}|{k}']  # noqa: E731
    dims, level = tuple(g('dims')), g('level')
    ds = xl.Dataset({k: (dims, g(k)) for k in (T, Z, Q)},
                    {'time': np.arange(2), 'level': level,
                     'latitude': np.linspace(-60, 60, 5),
                     'longitude': np.arange(8) * 45.0})
    lapse = dv.LapseRate().compute(ds).values
    np.testing.assert_array_equal(
        lapse, to.lapse_rate(g(T), g(Z), level, dims.index('level')))
    if level.dtype != np.float32:
      np.testing.assert_array_equal(lapse, g('lapse_rate'))
    rh = dv.RelativeHumidity().compute(ds).values
    p = _pressure(level, dims)
    _assert_rh(rh, g(T), g(Q), p)
    _, svp = to.relative_humidity(g(T), g(Q), p, with_svp=True)
    want = g('relative_humidity')
    ok = np.isnan(want) | (np.abs(rh - want) <= to.rh_bound(want, svp, p,
                                                            np.float32))
    assert ok.all(), name
  ds = xl.Dataset({T: (('level',), vec['metpy|temperature']),
                   Q: (('level',), vec['metpy|specific_humidity'])},
                  {'level': vec['metpy|level']})
  got = dv.RelativeHumidity().compute(ds).values
  assert got.dtype == np.float64
  np.testing.assert_allclose(got, vec['metpy|expected'], atol=1e-4)
  np.testing.assert_allclose(got, vec['metpy|relative_humidity'], rtol=1e-14)

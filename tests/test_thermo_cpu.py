"""CPU: the lapse rate and relative humidity.  tests/thermo_oracle.py is pinned
to np.gradient and NumPy's own expressions, and held to vectors from the
reference's own classes (tests/golden/make_thermo_vectors.py); the operator
layer runs end to end on `fake_ctx_thermo`, a NumPy interpretation of
wb2_lapse_rate and wb2_relative_humidity, in every layout, dtype and error
case."""
import os

import numpy as np
import pytest

import thermo_oracle as to

HERE = os.path.dirname(os.path.abspath(__file__))
T, Z, Q = 'temperature', 'geopotential', 'specific_humidity'
TLLL = ('time', 'level', 'latitude', 'longitude')
WB2_LEVELS = np.array([50, 100, 150, 200, 250, 300, 400, 500, 600, 700, 850,
                       925, 1000])
LAT, LON = np.linspace(-60, 60, 5), np.arange(8) * 45.0


def _height(level):
  return 44330.8 * (1 - (np.asarray(level, np.float64) / 1013.25) ** 0.190263)


def _fields(dims, level, seed, dtype=np.float32, nan=True):
  """Realistic temperature, geopotential and specific humidity profiles."""
  sizes = {'time': 2, 'level': len(level), 'latitude': LAT.size,
           'longitude': LON.size}
  shape = tuple(sizes[d] for d in dims)
  rs = np.random.RandomState(seed)
  prof = [None] * len(dims)
  prof[dims.index('level')] = slice(None)
  h = _height(level)[tuple(prof)]
  f = {T: (288.15 - 6.5e-3 * np.minimum(h, 11000) +
           rs.normal(scale=3, size=shape)).astype(dtype),
       Z: (9.81 * h + rs.normal(scale=40, size=shape)).astype(dtype),
       Q: (np.abs(rs.normal(scale=6e-3, size=shape)) *
           np.exp(-h / 2500)).astype(dtype)}
  if nan:
    f[T].reshape(-1)[3] = np.nan
    f[Z].reshape(-1)[7] = np.nan
    f[Q].reshape(-1)[1] = np.nan
  return f


def _dataset(xl, dims, fields, level, **extra):
  coords = {'time': np.arange(2), 'level': np.asarray(level),
            'latitude': LAT, 'longitude': LON}
  coords = {k: c for k, c in coords.items() if k in dims}
  coords.update(extra)
  return xl.Dataset({k: (dims, a) for k, a in fields.items()}, coords)


def _run(fn, *a, **kw):
  import fake_ctx_thermo
  with fake_ctx_thermo.installed() as fake:
    return fn(*a, **kw), fake


def _numpy_rh(t, q, p):
  """NumPy's own arithmetic of the reference's expression, on arrays."""
  with np.errstate(all='ignore'):
    vapour = 6.112 * np.exp(17.67 * (t - 273.15) / (t - 29.65))
    ratio = q / (1 - q)
    return ratio / (0.622 * vapour / (p - vapour))


def _pressure(level, dims, axis_dim='level'):
  shape = [1] * len(dims)
  shape[dims.index(axis_dim)] = -1
  return np.asarray(level).reshape(shape)


# -- the oracle against np.gradient and NumPy's expressions ---------------------
@pytest.mark.parametrize('level', [WB2_LEVELS, WB2_LEVELS[::-1], [500, 700, 900],
                                   [850, 1000], [100.0, 137.5, 300, 312.25]],
                         ids=['wb2', 'wb2_desc', 'uniform', 'two', 'float'])
@pytest.mark.parametrize('dtype', [np.float32, np.float64])
@pytest.mark.parametrize('axis', [0, 1, 2])
def test_oracle_gradient_is_np_gradient(level, dtype, axis):
  rs = np.random.RandomState(0)
  shape = [3, 4, 5]
  shape[axis] = len(level)
  f = (rs.normal(scale=1e3, size=shape) + 5e4).astype(dtype)
  f.reshape(-1)[2] = np.nan
  f.reshape(-1)[9] = np.inf
  with np.errstate(invalid='ignore'):
    want = np.gradient(f, np.asarray(level), axis=axis)
  got = to.gradient(f, level, axis)
  assert got.dtype == dtype
  np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize('dtype', [np.float32, np.float64])
def test_oracle_lapse_rate_is_numpy_arithmetic(dtype):
  f = _fields(TLLL, WB2_LEVELS, 0, dtype)
  f[Z][0, :, 0, 2] = f[Z][0, 0, 0, 2]  # dz == 0 in one column
  with np.errstate(all='ignore'):
    want = np.gradient(f[T], WB2_LEVELS, axis=1) / (
        (1 / 9.81) * np.gradient(f[Z], WB2_LEVELS, axis=1))
  got = to.lapse_rate(f[T], f[Z], WB2_LEVELS, 1)
  assert got.dtype == dtype
  np.testing.assert_array_equal(got, want)
  assert np.isinf(got[0, :, 0, 2]).any() or np.isnan(got[0, :, 0, 2]).all()


@pytest.mark.parametrize('level_dtype,dtype', [
    (np.int64, np.float32), (np.float32, np.float32), (np.int64, np.float64),
    (np.int16, np.float32), (np.float64, np.float32)])
def test_oracle_relative_humidity_is_numpy_arithmetic(level_dtype, dtype):
  f = _fields(TLLL, WB2_LEVELS, 1, dtype)
  p = _pressure(WB2_LEVELS.astype(level_dtype), TLLL)
  want = _numpy_rh(f[T], f[Q], p)
  got, svp = to.relative_humidity(f[T], f[Q], p, with_svp=True)
  assert got.dtype == want.dtype == np.result_type(level_dtype, dtype)
  # with NumPy's own exp in place of the rounded float64 one: bit for bit
  with np.errstate(all='ignore'):
    e = np.exp(to.bolton_argument(f[T]))
  np.testing.assert_array_equal(to.relative_humidity(f[T], f[Q], p, e=e), want)
  # and within the header's bound with it
  np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
  ok = np.isnan(want) | (np.abs(got - want) <= to.rh_bound(want, svp, p, dtype))
  assert ok.all()


def test_exp_gap_over_every_float32_temperature():
  """The header's measured gap: NumPy's float32 exp against exp evaluated in
  float64 and rounded once, over every float32 T in [180, 330] K."""
  t = np.arange(np.float32(180).view(np.int32),
                np.float32(330).view(np.int32) + 1,
                dtype=np.int32).view(np.float32)
  assert t.size == 7405569
  x = to.bolton_argument(t)
  ulp = np.abs(np.exp(x).view(np.int32).astype(np.int64) -
               to.bolton_exp(x).view(np.int32))
  assert ulp.max() <= 2
  p = np.float32(850)
  want = _numpy_rh(t, np.float32(5e-3), np.int64(850))
  got, svp = to.relative_humidity(t, np.full_like(t, 5e-3), np.int64(850),
                                  with_svp=True)
  assert (np.abs(got - want) <= to.rh_bound(want, svp, p, np.float32)).all()


# -- the oracle against the reference's own code --------------------------------
def _vectors():
  z = np.load(os.path.join(HERE, 'golden', 'reference_thermo_vectors.npz'))
  return z, sorted({k.split('|')[0] for k in z.files} - {'metpy'})


def test_oracle_matches_the_reference_vectors():
  vec, names = _vectors()
  assert len(names) == 5
  for name in names:
    g = lambda k: vec[f'{name}|{k}']  # noqa: E731
    dims, level = tuple(g('dims')), g('level')
    la = dims.index('level')
    lapse = to.lapse_rate(g(T), g(Z), level, la)
    want = g('lapse_rate')
    assert lapse.dtype == want.dtype == np.float32
    if level.dtype == np.float32:
      # the reference differences float32 levels, so its stencil weights and
      # ours differ in the last bits; in the dz == 0 column that decides
      # between an exact 0 (inf) and a tiny dz (a huge finite value)
      sane = (np.abs(lapse) < 1) & (np.abs(want) < 1)
      assert (~sane).sum() <= 2 * level.size + 4
      np.testing.assert_allclose(lapse[sane], want[sane], rtol=1e-5, atol=1e-7,
                                 err_msg=name)
    else:
      np.testing.assert_array_equal(lapse, want, err_msg=name)
    assert np.isinf(want).any() or np.isnan(want).sum() > 10  # the dz == 0 column
    p = _pressure(level, dims)
    rh, svp = to.relative_humidity(g(T), g(Q), p, with_svp=True)
    want = g('relative_humidity')
    assert rh.dtype == want.dtype == np.result_type(level.dtype, np.float32)
    np.testing.assert_array_equal(np.isnan(rh), np.isnan(want))
    ok = np.isnan(want) | (np.abs(rh - want) <= to.rh_bound(want, svp, p,
                                                            np.float32))
    assert ok.all(), name
  # derived_variables_test.py::testRelativeHumidity: integer temperature
  t, q, lev = vec['metpy|temperature'], vec['metpy|specific_humidity'], vec[
      'metpy|level']
  assert t.dtype == np.int64
  rh = to.relative_humidity(t, q, lev)
  assert rh.dtype == np.float64
  np.testing.assert_allclose(rh, vec['metpy|expected'], atol=1e-4)
  np.testing.assert_allclose(rh, vec['metpy|relative_humidity'], rtol=1e-14)


def test_operators_match_the_reference_vectors():
  from weatherbench2_b200 import derived_variables as dv, xarray_lite as xl
  vec, names = _vectors()
  for name in names:
    g = lambda k: vec[f'{name}|{k}']  # noqa: E731
    dims, level = tuple(g('dims')), g('level')
    ds = _dataset(xl, dims, {k: g(k) for k in (T, Z, Q)}, level)
    got, _ = _run(dv.LapseRate().compute, ds)
    assert got.dims == dims
    np.testing.assert_array_equal(
        got.values, to.lapse_rate(g(T), g(Z), level, dims.index('level')))
    if level.dtype != np.float32:
      np.testing.assert_array_equal(got.values, g('lapse_rate'))
    got, _ = _run(dv.RelativeHumidity().compute, ds)
    assert got.dims == dims and got.values.dtype == g('relative_humidity').dtype
    np.testing.assert_array_equal(
        got.values, to.relative_humidity(g(T), g(Q), _pressure(level, dims)))
  ds = xl.Dataset({T: (('level',), vec['metpy|temperature']),
                   Q: (('level',), vec['metpy|specific_humidity'])},
                  {'level': vec['metpy|level']})
  got, _ = _run(dv.RelativeHumidity().compute, ds)
  assert got.values.dtype == np.float64
  np.testing.assert_allclose(got.values, vec['metpy|expected'], atol=1e-4)


# -- the operator layer on the NumPy interpretation of the entries --------------
LAYOUTS = [TLLL, ('time', 'level', 'longitude', 'latitude'),
           ('level', 'time', 'latitude', 'longitude'),
           ('time', 'latitude', 'longitude', 'level'),
           ('longitude', 'level', 'time', 'latitude')]


@pytest.mark.parametrize('dims', LAYOUTS, ids=lambda d: '-'.join(x[:3] for x in d))
@pytest.mark.parametrize('dtype', [np.float32, np.float64])
def test_both_classes_in_every_layout(dims, dtype):
  from weatherbench2_b200 import derived_variables as dv, xarray_lite as xl
  level = WB2_LEVELS[3:10]
  f = _fields(dims, level, 2, dtype)
  ds = _dataset(xl, dims, f, level)
  la = dims.index('level')
  got, fake = _run(dv.LapseRate().compute, ds)
  assert got.dims == dims and got.values.dtype == dtype
  assert set(got.coords) == set(ds.coords)
  np.testing.assert_array_equal(got.values, to.lapse_rate(f[T], f[Z], level, la))
  nouter = int(np.prod([ds.sizes[d] for d in dims[:la]]))
  ninner = int(np.prod([ds.sizes[d] for d in dims[la + 1:]]))
  assert fake.calls == [('lapse_rate', int(dtype == np.float64), nouter,
                         level.size, ninner, False)]
  got, fake = _run(dv.RelativeHumidity().compute, ds)
  assert got.dims == dims and got.values.dtype == np.float64
  np.testing.assert_array_equal(
      got.values, to.relative_humidity(f[T], f[Q], _pressure(level, dims)))
  assert fake.calls[-1][3:] == (nouter, level.size, ninner)
  assert len(fake.calls) == 1


def test_operands_in_different_dim_orders():
  from weatherbench2_b200 import derived_variables as dv, xarray_lite as xl
  level = np.array([300, 500, 700, 850])
  f = _fields(TLLL, level, 3)
  perm = ('longitude', 'time', 'latitude', 'level')
  ax = tuple(TLLL.index(d) for d in perm)
  ds = _dataset(xl, TLLL, {T: f[T]}, level)
  for k in (Z, Q):
    ds[k] = xl.DataArray(np.ascontiguousarray(np.transpose(f[k], ax)), perm)
  got, _ = _run(dv.LapseRate().compute, ds)
  assert got.dims == TLLL  # temperature's
  np.testing.assert_array_equal(got.values, to.lapse_rate(f[T], f[Z], level, 1))
  got, _ = _run(dv.RelativeHumidity().compute, ds)
  assert got.dims == perm  # specific humidity's
  want = to.relative_humidity(f[T], f[Q], _pressure(level, TLLL))
  np.testing.assert_array_equal(got.values, np.transpose(want, ax))


@pytest.mark.parametrize('level_dtype,dtype,out', [
    (np.int64, np.float32, np.float64), (np.float32, np.float32, np.float32),
    (np.float64, np.float32, np.float64), (np.int64, np.float64, np.float64),
    (np.float32, np.float64, np.float64), (np.int16, np.float32, np.float32),
    (np.int64, np.int64, np.float64)])
def test_relative_humidity_output_dtype(level_dtype, dtype, out):
  from weatherbench2_b200 import derived_variables as dv, xarray_lite as xl
  level = np.array([300, 500, 850], level_dtype)
  f = _fields(TLLL, level, 4, np.float64, nan=False)
  f = {k: (np.round(a) if np.dtype(dtype).kind == 'i' and k == T else a
           ).astype(dtype) if k == T or np.dtype(dtype).kind != 'i' else a
       for k, a in f.items()}
  ds = _dataset(xl, TLLL, f, level)
  got, fake = _run(dv.RelativeHumidity().compute, ds)
  assert got.values.dtype == out
  want = to.relative_humidity(f[T], f[Q], _pressure(level, TLLL))
  assert want.dtype == out
  np.testing.assert_array_equal(got.values, want)
  code = int(np.dtype(dtype).kind == 'i' or dtype == np.float64)
  assert fake.calls[-1][1:3] == (code, int(out == np.float64))


def test_scalar_and_other_pressure_coordinates():
  from weatherbench2_b200 import derived_variables as dv, xarray_lite as xl
  dims = ('time', 'latitude', 'longitude')
  f = _fields(('time', 'level', 'latitude', 'longitude'), [500], 5)
  f = {k: a[:, 0] for k, a in f.items()}
  # a scalar `level` coordinate: one pressure for every cell
  ds = xl.Dataset({k: (dims, a) for k, a in f.items()},
                  {'time': np.arange(2), 'latitude': LAT, 'longitude': LON,
                   'level': np.array(500)})
  got, fake = _run(dv.RelativeHumidity().compute, ds)
  assert got.dims == dims and got.values.dtype == np.float64
  np.testing.assert_array_equal(
      got.values, to.relative_humidity(f[T], f[Q], np.array(500)))
  assert fake.calls[-1][3:] == (1, 1, f[T].size)
  np.testing.assert_array_equal(got.coords['level'].values, 500)
  # pressure_name naming a float32 coordinate along `level`
  level = np.array([300, 500, 850])
  g = _fields(TLLL, level, 6)
  pres = np.array([301.5, 498.25, 851], np.float32)
  ds = _dataset(xl, TLLL, g, level,
                pressure=xl.Coord(('level',), pres))
  got, _ = _run(dv.RelativeHumidity(pressure_name='pressure').compute, ds)
  assert got.values.dtype == np.float32
  np.testing.assert_array_equal(
      got.values, to.relative_humidity(g[T], g[Q], _pressure(pres, TLLL)))
  # pressure_name naming a coordinate along another dim of the data
  plat = np.linspace(900, 1000, LAT.size)
  ds = _dataset(xl, TLLL, g, level, plat=xl.Coord(('latitude',), plat))
  got, fake = _run(dv.RelativeHumidity(pressure_name='plat').compute, ds)
  np.testing.assert_array_equal(got.values, to.relative_humidity(
      g[T], g[Q], _pressure(plat, TLLL, 'latitude')))
  assert fake.calls[-1][3:] == (2 * 3, LAT.size, LON.size)


def test_torch_cpu_input_gives_numpy():
  torch = pytest.importorskip('torch')
  from weatherbench2_b200 import derived_variables as dv, xarray_lite as xl
  level = np.array([300, 500, 850])
  f = _fields(TLLL, level, 7)
  ds = _dataset(xl, TLLL, {k: torch.from_numpy(a) for k, a in f.items()}, level)
  got, _ = _run(dv.LapseRate().compute, ds)
  assert isinstance(got.values, np.ndarray)
  np.testing.assert_array_equal(got.values, to.lapse_rate(f[T], f[Z], level, 1))
  got, _ = _run(dv.RelativeHumidity().compute, ds)
  assert isinstance(got.data, np.ndarray)


def test_class_fields_match_the_reference():
  from weatherbench2_b200 import derived_variables as dv
  lr, rh = dv.LapseRate(), dv.RelativeHumidity()
  assert isinstance(lr, dv.DerivedVariable) and isinstance(rh, dv.DerivedVariable)
  assert (lr.temperature_name, lr.geopotential_name) == (T, Z)
  assert lr.base_variables == [T, Z]
  assert lr.core_dims == ((['level'], ['level']), ['level'])
  assert (rh.temperature_name, rh.specific_humidity_name,
          rh.pressure_name) == (T, Q, 'level')
  assert rh.base_variables == [T, Q, 'level']
  assert rh.core_dims == (([], []), [])
  assert dv.RelativeHumidity(pressure_name='p').base_variables == [T, Q, 'p']
  for name in ('lapse_rate', 'relative_humidity'):
    assert name not in dv.DERIVED_VARIABLE_DICT


def test_errors():
  from weatherbench2_b200 import derived_variables as dv, xarray_lite as xl
  level = np.array([300, 500, 850])
  f = _fields(TLLL, level, 8)
  ds = _dataset(xl, TLLL, f, level)
  for var in (dv.LapseRate(geopotential_name='z'),
              dv.RelativeHumidity(specific_humidity_name='q'),
              dv.RelativeHumidity(pressure_name='pressure')):
    with pytest.raises(KeyError):  # a missing base variable or coordinate
      _run(var.compute, ds)
  flat = xl.Dataset({k: (('time', 'latitude', 'longitude'), a[:, 0])
                     for k, a in f.items()},
                    {'latitude': LAT, 'longitude': LON,
                     'level': xl.Coord(('level',), level)})
  with pytest.raises(ValueError):  # no level dimension
    _run(dv.LapseRate().compute, flat)
  with pytest.raises(ValueError):  # the pressure lies along a dim q lacks
    _run(dv.RelativeHumidity().compute, flat)
  no_coord = xl.Dataset({k: (TLLL, a) for k, a in f.items()},
                        {'latitude': LAT, 'longitude': LON})
  with pytest.raises(ValueError):  # no level coordinate
    _run(dv.LapseRate().compute, no_coord)
  with pytest.raises(KeyError):
    _run(dv.RelativeHumidity().compute, no_coord)
  one = _dataset(xl, TLLL, {k: a[:, :1] for k, a in f.items()}, level[:1])
  with pytest.raises(ValueError):  # fewer than 2 levels
    _run(dv.LapseRate().compute, one)
  other = _dataset(xl, TLLL, f, level)
  other[Z] = xl.DataArray(f[Z][0], TLLL[1:])
  other[Q] = xl.DataArray(f[Q][0], TLLL[1:])
  for var in (dv.LapseRate(), dv.RelativeHumidity()):
    with pytest.raises(ValueError):  # dims differ
      _run(var.compute, other)
  two_d = _dataset(xl, TLLL, f, level,
                   p2=xl.Coord(('level', 'latitude'),
                               np.ones((3, LAT.size))))
  with pytest.raises(ValueError):  # a two-dimensional pressure coordinate
    _run(dv.RelativeHumidity(pressure_name='p2').compute, two_d)
  for bad in (np.float16, np.bool_):
    g = dict(f, **{T: f[T].astype(bad)})
    for var in (dv.LapseRate(), dv.RelativeHumidity()):
      with pytest.raises(TypeError, match=T):
        _run(var.compute, _dataset(xl, TLLL, g, level))
  # the entries reject what the operators never send
  import fake_ctx_thermo
  from weatherbench2_b200 import _lib
  ctx = fake_ctx_thermo.ThermoFakeContext()
  with pytest.raises(_lib.Wb2Error):
    ctx.lapse_rate(7, 0, 0, 1, 3, 1, np.zeros((3, 3)), False, 0)


def test_both_classes_in_evaluate_in_memory(tmp_path):
  """MSE of the derived lapse rate and relative humidity through
  evaluate_in_memory equals the same evaluation fed the oracle's values as
  plain variables."""
  from test_evaluation_gpu import _mock
  from weatherbench2_b200 import config, derived_variables as dv, evaluation
  from weatherbench2_b200 import metrics, xarray_lite as xl
  level = (500, 700, 850)
  fc, truth, fv, tv, _, _, fdims, tdims = _mock(
      nlat=9, nlon=12, levels=level, variables=(T, Z, Q))
  for arrays in (fv, tv):  # realistic magnitudes, in place
    arrays[T] *= 4
    arrays[T] += 260
    arrays[Z] *= 300
    arrays[Z] += 9.81 * _height(level)[:, None, None]
    np.abs(arrays[Q], out=arrays[Q])
    arrays[Q] *= 4e-3
  derived = {'lapse_rate': dv.LapseRate(),
             'relative_humidity': dv.RelativeHumidity()}

  def config_for(f, t, variables, derived_variables):
    dc = config.Data(
        selection=config.Selection(variables=variables,
                                   time_slice=slice(None, None)),
        paths=config.Paths(forecast=f, obs=t, output_dir=str(tmp_path)),
        by_init=True)
    ec = {'det': config.Eval(metrics={'mse': metrics.MSE()},
                             derived_variables=derived_variables)}
    return dc, ec

  dc, ec = config_for(fc, truth, [T], derived)
  out, fake = _run(evaluation.evaluate_in_memory, dc, ec)
  assert {c[0] for c in fake.calls} >= {'lapse_rate', 'relative_humidity'}

  def plain(ds, arrays, dims):
    la = dims.index('level')
    p = _pressure(np.array(level), dims)
    return xl.Dataset(
        {T: (dims, arrays[T]),
         'lapse_rate': (dims, to.lapse_rate(arrays[T], arrays[Z], level, la)),
         'relative_humidity': (dims, to.relative_humidity(arrays[T], arrays[Q],
                                                          p))},
        {k: c for k, c in ds.coords.items()})

  dc, ec = config_for(plain(fc, fv, fdims), plain(truth, tv, tdims),
                      [T, 'lapse_rate', 'relative_humidity'], {})
  want, _ = _run(evaluation.evaluate_in_memory, dc, ec)
  for k in ('lapse_rate', 'relative_humidity'):
    got = np.asarray(out['det'][k].values)
    np.testing.assert_array_equal(got, np.asarray(want['det'][k].values),
                                  err_msg=k)
    assert np.isfinite(got).all()

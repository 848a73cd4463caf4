"""CPU: the column integrals (total column water, integrated water transport,
eddy kinetic energy).  tests/column_oracle.py is held to hand answers and to
vectors from the reference's own classes (tests/golden/make_column_vectors.py);
the operator layer runs end to end on `fake_ctx_column`, a NumPy
interpretation of wb2_column_integral, in every layout and error case."""
import os

import numpy as np
import pytest

import column_oracle as co

HERE = os.path.dirname(os.path.abspath(__file__))
Q, U, V = 'specific_humidity', 'u_component_of_wind', 'v_component_of_wind'
TLLL = ('time', 'level', 'latitude', 'longitude')
COLUMN_NAMES = ('total_column_vapor', 'total_column_liquid', 'total_column_ice',
                'integrated_vapor_transport', 'eddy_kinetic_energy')


def _dataset(xl, dims, fields, level, lat, lon, ntime=2):
  coords = {'time': np.arange(ntime), 'level': np.asarray(level),
            'latitude': lat, 'longitude': lon}
  return xl.Dataset({k: (dims, a) for k, a in fields.items()},
                    {k: c for k, c in coords.items() if k in dims})


def _fields(shape, seed, dtype=np.float32, nan=True):
  rs = np.random.RandomState(seed)
  q = np.abs(rs.normal(scale=4e-3, size=shape)).astype(dtype)
  u = (5 + rs.normal(scale=12, size=shape)).astype(dtype)
  v = rs.normal(scale=8, size=shape).astype(dtype)
  if nan:
    q.reshape(-1)[2] = np.nan
    u.reshape(-1)[shape[-1] + 1] = np.nan
  return {Q: q, U: u, V: v}


def _run(fn, *a, **kw):
  import fake_ctx_column
  with fake_ctx_column.installed() as fake:
    return fn(*a, **kw), fake


def _want(kind, dims, f, level, **kw):
  la = dims.index('level')
  if kind == 'tc':
    r = co.total_column(f[Q], level, la)
  elif kind == 'ivt':
    r = co.ivt(f[Q], f[U], f[V], level, la, **kw)
  else:
    r = co.eke(f[U], f[V], level, la, dims.index('longitude'))
  return r


# -- the oracle against hand answers --------------------------------------------
def test_q_linear_in_pressure_integrates_exactly():
  level = np.array([100, 250, 300, 500, 850, 1000])
  q = (2e-3 + 1e-6 * level).astype(np.float64)[:, None]
  got = co.total_column(q, level)
  exact = (2e-3 * (1000 - 100) + 0.5e-6 * (1000 ** 2 - 100 ** 2)) / 9.81
  np.testing.assert_allclose(got, exact, rtol=1e-14)


@pytest.mark.parametrize('level', [(50, 300, 1000), (1000, 700, 250, 50)])
def test_constant_field(level):
  c = np.float32(3e-3)
  got = co.total_column(np.full((len(level), 4), c), level)
  np.testing.assert_allclose(got, float(c) * (level[-1] - level[0]) / 9.81,
                             rtol=1e-15)


def test_zonally_uniform_wind_has_no_eddy_kinetic_energy():
  rs = np.random.RandomState(0)
  u = np.repeat(rs.normal(size=(4, 3, 1)), 16, axis=2).astype(np.float32)
  v = np.repeat(rs.normal(size=(4, 3, 1)), 16, axis=2).astype(np.float32)
  assert (co.eke(u, v, (100, 500, 850, 1000), 0, 2) == 0).all()


def test_eddy_kinetic_energy_of_a_zonal_wave():
  nlon, m, a = 64, 3, 7.0
  lam = np.arange(nlon) * 2 * np.pi / nlon
  level = np.array([200, 500, 850, 1000])
  u = np.broadcast_to(a * np.cos(m * lam), (level.size, 2, nlon))
  got = co.eke(u, np.zeros_like(u), level, 0, 2)
  want = 0.5 * a * a * np.cos(m * lam) ** 2 * (level[-1] - level[0])
  np.testing.assert_allclose(got, np.broadcast_to(want, got.shape),
                             rtol=1e-12, atol=1e-9)


# -- the oracle against the reference's own code --------------------------------
def _vectors():
  z = np.load(os.path.join(HERE, 'golden', 'reference_column_vectors.npz'))
  return z, sorted({k.split('|')[0] for k in z.files})


IVT_WINDOWS = {'integrated_vapor_transport': (300, 1000),
               'ivt_all_levels': (None, None), 'ivt_narrow': (500, 850),
               'ivt_empty': (1000, 300)}
SPECIES = {'total_column_vapor': Q,
           'total_column_liquid': 'specific_cloud_liquid_water_content',
           'total_column_ice': 'specific_cloud_ice_water_content'}


def _oracle_for(vec, name, kind):
  dims = tuple(vec[f'{name}|dims'])
  level = vec[f'{name}|level']
  la, lo = dims.index('level'), dims.index('longitude')
  g = lambda k: vec[f'{name}|{k}']  # noqa: E731
  if kind in SPECIES:
    y = g(SPECIES[kind])
    return co.total_column(y, level, la), co.INV_G * co.sum_bound(y, level, la)
  if kind in IVT_WINDOWS:
    lmin, lmax = IVT_WINDOWS[kind]
    r = co.ivt(g(Q), g(U), g(V), level, la, lmin, lmax)
    sl = co.window(level, lmin, lmax)
    take = lambda a: np.moveaxis(a, la, 0)[sl]  # noqa: E731
    b = co.INV_G * (co.sum_bound(take(g(Q)) * take(g(U)), level[sl]) +
                    co.sum_bound(take(g(Q)) * take(g(V)), level[sl]))
    return r, b + 2.0 ** -50 * np.abs(r)
  return (co.eke(g(U), g(V), level, la, lo),
          co.eke_bound(g(U), g(V), level, la, lo))


def test_oracle_matches_the_reference_run_vectors():
  vec, names = _vectors()
  assert len(names) == 7
  kinds = list(SPECIES) + list(IVT_WINDOWS) + ['eddy_kinetic_energy']
  for name in names:
    innermost = tuple(vec[f'{name}|dims'])[-1] == 'level'
    for kind in kinds:
      want = vec[f'{name}|{kind}']
      got, bound = _oracle_for(vec, name, kind)
      assert want.dtype == np.float64
      np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
      if kind == 'eddy_kinetic_energy' or innermost:
        ok = np.isnan(want) | (np.abs(got - want) <= bound)
        assert ok.all(), (name, kind, np.nanmax(np.abs(got - want) - bound))
      else:  # the same summation order: bit for bit
        np.testing.assert_array_equal(got, want, err_msg=f'{name} {kind}')
  # pandas leaves the descending slice empty: the reference integrates nothing
  assert (vec['descending|integrated_vapor_transport'] == 0).all()
  assert (vec['ascending|ivt_empty'] == 0).all()
  assert (vec['single_level|total_column_vapor'] == 0).all()


def test_operators_match_the_reference_run_vectors():
  from weatherbench2_b200 import derived_variables as dv, xarray_lite as xl
  vec, names = _vectors()
  for name in names:
    dims = tuple(vec[f'{name}|dims'])
    fields = {k.split('|')[1]: vec[k] for k in vec.files
              if k.startswith(name + '|') and vec[k].ndim == len(dims)
              and vec[k].dtype == np.float32}
    ds = _dataset(xl, dims, fields, vec[f'{name}|level'],
                  vec[f'{name}|latitude'], vec[f'{name}|longitude'])
    for kind in list(SPECIES) + list(IVT_WINDOWS) + ['eddy_kinetic_energy']:
      var = (dv.IntegratedWaterTransport(*(), level_min=IVT_WINDOWS[kind][0],
                                         level_max=IVT_WINDOWS[kind][1])
             if kind in IVT_WINDOWS else dv.DERIVED_VARIABLE_DICT[kind])
      got, _ = _run(var.compute, ds)
      assert got.dims == tuple(d for d in dims if d != 'level')
      want, _ = _oracle_for(vec, name, kind)
      np.testing.assert_array_equal(got.values, co.rounded(want, np.float32),
                                    err_msg=f'{name} {kind}')


# -- the operator layer on the NumPy interpretation of the entry ----------------
LAT, LON = np.linspace(-90, 90, 7), np.arange(10) * 36.0


@pytest.mark.parametrize('dims', [
    TLLL, ('time', 'level', 'longitude', 'latitude'),
    ('level', 'time', 'latitude', 'longitude'),
    ('latitude', 'level', 'time', 'longitude'),
    ('time', 'latitude', 'longitude', 'level'),
    ('longitude', 'time', 'level', 'latitude')],
                         ids=lambda d: '-'.join(x[:3] for x in d))
@pytest.mark.parametrize('dtype', [np.float32, np.float64])
def test_every_class_in_every_layout(dims, dtype):
  from weatherbench2_b200 import derived_variables as dv, xarray_lite as xl
  level = (200, 300, 500, 700, 850, 1000)
  shape = tuple({'time': 2, 'level': 6, 'latitude': 7, 'longitude': 10}[d]
                for d in dims)
  f = _fields(shape, 1, dtype)
  ds = _dataset(xl, dims, f, level, LAT, LON)
  out_dims = tuple(d for d in dims if d != 'level')
  for kind, var in (('tc', dv.TotalColumnWater()),
                    ('ivt', dv.IntegratedWaterTransport(level_min=300,
                                                        level_max=850)),
                    ('eke', dv.EddyKineticEnergy())):
    got, fake = _run(var.compute, ds)
    assert got.dims == out_dims and got.values.dtype == dtype, kind
    assert set(got.coords) == {d for d in out_dims if d != 'time'} | (
        {'time'} if 'time' in dims else set())
    kw = dict(level_min=300, level_max=850) if kind == 'ivt' else {}
    want = co.rounded(_want(kind, dims, f, level, **kw), dtype)
    if kind == 'eke' and dtype == np.float64:  # the zonal sum's order
      np.testing.assert_allclose(got.values, want, rtol=1e-13, err_msg=kind)
    else:
      np.testing.assert_array_equal(got.values, want, err_msg=kind)
    call = fake.calls[-1]
    assert call[0] == 'column_integral' and len(fake.calls) == 1
    if kind == 'ivt':  # levels 300..850: an offset of 1 and a count of 4
      assert call[5] == 4
    if kind == 'eke':
      lon_contig = dims.index('latitude') < dims.index('longitude')
      assert call[7:] == (10, 1 if lon_contig else 7)


def test_ivt_inputs_take_their_common_dtype_and_order():
  from weatherbench2_b200 import derived_variables as dv, xarray_lite as xl
  level = (300, 500, 850, 1000)
  f = _fields((2, 4, 7, 10), 2)
  f[U] = f[U].astype(np.float64)
  ds = _dataset(xl, TLLL, {Q: f[Q], V: f[V]}, level, LAT, LON)
  ds[U] = xl.DataArray(np.ascontiguousarray(np.transpose(f[U], (3, 0, 2, 1))),
                       ('longitude', 'time', 'latitude', 'level'))
  got, _ = _run(dv.IntegratedWaterTransport().compute, ds)
  assert got.values.dtype == np.float64
  want = co.ivt(f[Q], f[U], f[V], level, 1)
  np.testing.assert_array_equal(got.values, co.rounded(want, np.float64))


@pytest.mark.parametrize('level', [(500,), (1000, 850, 500, 300, 100)])
def test_single_level_and_descending_levels(level):
  from weatherbench2_b200 import derived_variables as dv, xarray_lite as xl
  f = _fields((2, len(level), 7, 10), 3)
  ds = _dataset(xl, TLLL, f, level, LAT, LON)
  ivt, fake = _run(dv.IntegratedWaterTransport().compute, ds)
  # one level inside the window, or none: descending levels empty the slice
  assert (ivt.values == 0).all() and fake.calls[-1][5] == (len(level) == 1)
  tc, _ = _run(dv.TotalColumnWater().compute, ds)
  eke, _ = _run(dv.EddyKineticEnergy().compute, ds)
  if len(level) == 1:
    assert (tc.values == 0).all() and (eke.values == 0).all()
  else:  # descending: the integral is negative, as trapz gives
    want = co.rounded(co.total_column(f[Q], level, 1), np.float32)
    np.testing.assert_array_equal(tc.values, want)
    assert np.nanmax(tc.values) < 0


def test_torch_cpu_and_lazily_gathered_input_give_numpy():
  torch = pytest.importorskip('torch')
  from weatherbench2_b200 import derived_variables as dv, xarray_lite as xl
  level = (300, 500, 850)
  f = _fields((2, 3, 7, 10), 4)
  ds = _dataset(xl, TLLL, {k: torch.from_numpy(a) for k, a in f.items()},
                level, LAT, LON)
  got, _ = _run(dv.TotalColumnWater().compute, ds)
  assert isinstance(got.values, np.ndarray)
  np.testing.assert_array_equal(
      got.values, co.rounded(co.total_column(f[Q], level, 1), np.float32))


def test_class_fields_match_the_reference():
  from weatherbench2_b200 import derived_variables as dv
  d = dv.DERIVED_VARIABLE_DICT
  for name in COLUMN_NAMES:
    assert name in d
  assert d['total_column_vapor'].base_variables == [Q]
  assert d['total_column_liquid'].base_variables == [
      'specific_cloud_liquid_water_content']
  assert d['total_column_ice'].base_variables == [
      'specific_cloud_ice_water_content']
  assert d['total_column_vapor'].core_dims == ((['level'],), [])
  ivt = d['integrated_vapor_transport']
  assert ivt.base_variables == [U, V, Q]
  assert (ivt.level_min, ivt.level_max) == (300, 1000)
  assert ivt.core_dims == ((['level'], ['level']), [])
  eke = d['eddy_kinetic_energy']
  assert isinstance(eke, dv._3DWindVariable)  # pylint: disable=protected-access
  assert eke.base_variables == [U, V]
  assert eke.core_dims == ((['level', 'longitude'], ['level', 'longitude']),
                           ['longitude'])
  assert dv.TotalColumnWater().water_species_name == Q
  for name in ('lapse_rate', 'relative_humidity'):
    with pytest.raises(KeyError):
      d[name]  # pylint: disable=pointless-statement


def test_errors():
  from weatherbench2_b200 import derived_variables as dv, xarray_lite as xl
  level = (300, 500, 850)
  f = _fields((2, 3, 7, 10), 5)
  ds = _dataset(xl, TLLL, f, level, LAT, LON)
  with pytest.raises(KeyError):  # a missing base variable
    _run(dv.TotalColumnWater('specific_cloud_ice_water_content').compute, ds)
  flat = _dataset(xl, ('time', 'latitude', 'longitude'),
                  {k: a[:, 0] for k, a in f.items()}, level, LAT, LON)
  for var in (dv.TotalColumnWater(), dv.IntegratedWaterTransport(),
              dv.EddyKineticEnergy()):
    with pytest.raises(ValueError):  # no level dimension
      _run(var.compute, flat)
  no_coord = xl.Dataset({k: (TLLL, a) for k, a in f.items()},
                        {'latitude': LAT, 'longitude': LON})
  for var in (dv.TotalColumnWater(), dv.IntegratedWaterTransport(),
              dv.EddyKineticEnergy()):
    with pytest.raises(KeyError):  # no level coordinate
      _run(var.compute, no_coord)
  other = _dataset(xl, TLLL, f, level, LAT, LON)
  other[U] = xl.DataArray(f[U][0], TLLL[1:])
  with pytest.raises(ValueError):  # dims differ
    _run(dv.EddyKineticEnergy().compute, other)
  for bad in (np.float16, np.int32):
    g = dict(f, **{U: f[U].astype(bad)})
    with pytest.raises(TypeError, match=U):
      _run(dv.IntegratedWaterTransport().compute,
           _dataset(xl, TLLL, g, level, LAT, LON))
  g = dict(f, **{Q: f[Q].astype(np.float16)})
  with pytest.raises(TypeError, match=Q):
    _run(dv.TotalColumnWater().compute, _dataset(xl, TLLL, g, level, LAT, LON))
  shuffled = _dataset(xl, TLLL, f, (500, 300, 850), LAT, LON)
  with pytest.raises(KeyError):  # not monotonic under IVT's slice
    _run(dv.IntegratedWaterTransport().compute, shuffled)
  # the other two do not slice, so they take any order
  got, _ = _run(dv.TotalColumnWater().compute, shuffled)
  np.testing.assert_array_equal(got.values, co.rounded(
      co.total_column(f[Q], (500, 300, 850), 1), np.float32))
  no_lon = _dataset(xl, ('time', 'level', 'latitude'),
                    {k: a[..., 0] for k, a in f.items()}, level, LAT, LON)
  with pytest.raises(ValueError):
    _run(dv.EddyKineticEnergy().compute, no_lon)


def test_ivt_and_eke_in_the_metric_loop():
  """MSE over the derived IVT and EKE equals the same loop fed the oracle's
  values as plain variables."""
  from weatherbench2_b200 import config, derived_variables as dv, evaluation
  from weatherbench2_b200 import metrics, regions, xarray_lite as xl
  level = (250, 300, 500, 700, 850, 925, 1000)
  f = _fields((3, 7, 7, 10), 6, nan=False)
  t = _fields((3, 7, 7, 10), 7, nan=False)
  fds = _dataset(xl, TLLL, f, level, LAT, LON, ntime=3)
  tds = _dataset(xl, TLLL, t, level, LAT, LON, ntime=3)
  names = ('integrated_vapor_transport', 'eddy_kinetic_energy')
  ms = {'mse': metrics.MSE()}
  rg = {'global': regions.SliceRegion(), 'tropics': regions.SliceRegion(
      lat_slice=slice(-30, 30))}
  ec = config.Eval(metrics=ms, regions=rg, derived_variables={
      k: dv.DERIVED_VARIABLE_DICT[k] for k in names})
  res, fake = _run(evaluation._metric_and_region_loop, fds, tds, ec,  # pylint: disable=protected-access
                   skipna=False)
  assert sum(c[0] == 'column_integral' for c in fake.calls) == 4
  d2 = ('time', 'latitude', 'longitude')

  def plain(x):
    return xl.Dataset(
        {'integrated_vapor_transport': (d2, co.rounded(
            _want('ivt', TLLL, x, level), np.float32)),
         'eddy_kinetic_energy': (d2, co.rounded(
             _want('eke', TLLL, x, level), np.float32))},
        {'time': np.arange(3), 'latitude': LAT, 'longitude': LON})

  want, _ = _run(evaluation._metric_and_region_loop, plain(f), plain(t),  # pylint: disable=protected-access
                 config.Eval(metrics=ms, regions=rg), skipna=False)
  for k in names:
    np.testing.assert_array_equal(np.asarray(res[k].values),
                                  np.asarray(want[k].values), err_msg=k)
    assert np.isfinite(np.asarray(res[k].values)).all()

"""Wind dynamics derived variables without a GPU: the float64 oracle
(tests/dynamics_oracle.py) pinned to hand-derived answers and to vectors from
the reference's own derived_variables.py (golden/make_dynamics_vectors.py),
and the operator layer end to end on `fake_ctx_dynamics` (NumPy interpreting
the wb2_wind_dynamics arguments): both layouts, both latitude orders, a
regional grid, levels both ways, every class in the metric loop, a by-init
evaluation and the errors.  tests/test_wind_dynamics_gpu.py runs the kernels."""
import os

import numpy as np
import pytest

import dynamics_cases as dc
import dynamics_oracle as do

HERE = os.path.dirname(os.path.abspath(__file__))
R = do.EARTH_RADIUS_M
M = do.METERS_PER_DEGREE
DIMS = ('latitude', 'longitude')


def _grid(nlat=19, nlon=24):
  return np.linspace(-90, 90, nlat), np.arange(nlon) * (360 / nlon)


def _f32(want):
  return np.asarray(want).astype(np.float32)


# -- the oracle against hand-derived answers ----------------------------------
def test_linear_fields_are_differentiated_exactly_including_the_edges():
  lat, lon = _grid()
  lon2, lat2 = np.meshgrid(lon, lat)
  u = (3.0 * lon2).astype(np.float32)   # d/dlon = 3 per degree, exactly
  v = (2.0 * lat2).astype(np.float32)   # d/dlat = 2 per degree, exactly
  cos = np.cos(np.deg2rad(lat))[:, None]
  dx = np.broadcast_to(np.where(cos > 1e-6, 3.0 / cos / M, 0.0), u.shape)
  dy = np.float32(2.0) / np.float32(M)
  div = do.compute('divergence', DIMS, lat, lon, u=u, v=v)
  np.testing.assert_array_equal(div, dx + np.float64(dy))
  assert (div[0] == dy).all() and (div[-1] == dy).all()  # poles: _d_dx = 0
  vort = do.compute('vorticity', DIMS, lat, lon, u=v, v=u)
  np.testing.assert_array_equal(vort, dx - np.float64(dy))


def test_solid_body_rotation_has_no_divergence_and_a_flat_vorticity():
  """u = U cos(lat), v = 0: divergence 0; vorticity -_d_dy(u) tends to
  U sin(lat) / R -- not the spherical 2 U sin(lat) / R, because the
  reference's _curl has no metric term."""
  U = 20.0
  for n in (181, 721, 2881):
    lat, lon = np.linspace(-90, 90, n), np.arange(8) * 45.0
    u = np.repeat((U * np.cos(np.deg2rad(lat)))[:, None], 8, 1)
    v = np.zeros_like(u)
    assert (do.compute('divergence', DIMS, lat, lon, u=u, v=v) == 0).all()
    vort = do.compute('vorticity', DIMS, lat, lon, u=u, v=v)[1:-1, 0]
    want = U * np.sin(np.deg2rad(lat[1:-1])) / R
    err = np.max(np.abs(vort - want)) / (U / R)
    assert err < 3e-4 * (181 / n)**2, (n, err)   # second order in the spacing
  assert np.max(np.abs(vort - 2 * want)) > 0.9 * U / R


def test_geostrophic_wind_of_a_known_stream_function():
  """z = f0 * psi with psi = -Ug * y + Vg * x (x, y in metres along the
  axes) gives u_geo = Ug f0 / f, v_geo = Vg f0 / (f cos(lat))."""
  lat, lon = np.linspace(20, 70, 11), np.linspace(0, 50, 11)
  f0, ug, vg = 1e-4, 12.0, -7.0
  lon2, lat2 = np.meshgrid(lon, lat)
  z = f0 * (-ug * lat2 * M + vg * lon2 * M)
  f = 2 * do.OMEGA * np.sin(np.deg2rad(lat))[:, None]
  cos = np.cos(np.deg2rad(lat))[:, None]
  u = do.compute('u_component_of_geostrophic_wind', DIMS, lat, lon, z=z)
  v = do.compute('v_component_of_geostrophic_wind', DIMS, lat, lon, z=z)
  np.testing.assert_allclose(u, np.broadcast_to(ug * f0 / f, u.shape),
                             rtol=1e-12)
  np.testing.assert_allclose(v, np.broadcast_to(vg * f0 / f / cos, v.shape),
                             rtol=1e-12)
  s = do.compute('geostrophic_wind_speed', DIMS, lat, lon, z=z)
  np.testing.assert_allclose(s, np.hypot(u, v), rtol=1e-15)
  # a wind equal to the geostrophic one has no ageostrophic part
  a = do.compute('ageostrophic_wind_speed', DIMS, lat, lon, u=u, v=v, z=z)
  assert np.max(a) < 1e-12 * np.max(s)


def test_equator_and_pole_rows():
  lat, lon = _grid(9, 8)
  lon2, lat2 = np.meshgrid(lon, lat)
  z = (5.0 * lat2 + 1.0 * np.minimum(lon2, 100)).astype(np.float32)
  z[0, 3] = np.nan  # NaN on the south pole row
  u = do.compute('u_component_of_geostrophic_wind', DIMS, lat, lon, z=z)
  v = do.compute('v_component_of_geostrophic_wind', DIMS, lat, lon, z=z)
  eq = 4
  assert lat[eq] == 0
  assert (u[eq] == -np.inf).all()             # -(5 / M) / 0
  assert (v[eq][lon < 150] == np.inf).all()   # (1 / cos / M) / 0
  assert np.isnan(v[eq][lon > 150]).all()     # 0 / 0 where z is flat
  assert (v[0] == 0).all() and (v[-1] == 0).all()  # _d_dx zeroed at poles
  assert np.isnan(u[0, 3]) and np.isnan(u[1, 3])   # _d_dy does see the NaN
  assert np.isfinite(np.delete(u, eq, 0)[:, [0, 1, 2, 4, 5, 6, 7]]).all()


# -- the oracle against the reference's own code --------------------------------
def _vectors():
  z = np.load(os.path.join(HERE, 'golden', 'reference_dynamics_vectors.npz'))
  names = sorted({k.split('|')[0] for k in z.files})
  return z, names


def test_oracle_matches_the_reference_run_vectors():
  vec, names = _vectors()
  assert len(names) == 5
  for name in names:
    dims = tuple(vec[f'{name}|dims'])
    args = dict(u=vec[f'{name}|u'], v=vec[f'{name}|v'], z=vec[f'{name}|z'],
                level=vec[f'{name}|level'])
    for kind in do.KINDS:
      want = vec[f'{name}|{kind}']
      got = do.compute(kind, dims, vec[f'{name}|latitude'],
                       vec[f'{name}|longitude'], **args)
      np.testing.assert_allclose(got, want, rtol=1e-12, atol=0,
                                 equal_nan=True, err_msg=f'{name} {kind}')
      assert (np.isinf(got) == np.isinf(want)).all(), (name, kind)


def test_operators_match_the_reference_run_vectors():
  from weatherbench2_b200 import derived_variables as dv, xarray_lite as xl
  import fake_ctx_dynamics
  vec, names = _vectors()
  for name in names:
    dims = tuple(vec[f'{name}|dims'])
    lat, lon = vec[f'{name}|latitude'], vec[f'{name}|longitude']
    data = {k: vec[f'{name}|{k}'] for k in 'uvz'}
    ds = dc.dataset(xl, dims, lat, lon, data, vec[f'{name}|level'], ntime=1)
    with fake_ctx_dynamics.installed():
      for kind in do.KINDS:
        got = dv.DERIVED_VARIABLE_DICT[kind].compute(ds)
        assert got.dims == dims
        np.testing.assert_array_equal(got.values, _f32(vec[f'{name}|{kind}']),
                                      err_msg=f'{name} {kind}')


# -- the operator layer on the NumPy interpretation of the entry ----------------
def _run(fn, *a, **kw):
  import fake_ctx_dynamics
  with fake_ctx_dynamics.installed() as fake:
    return fn(*a, **kw), fake


@pytest.mark.parametrize('grid', ['nonuniform32', 'descending', 'regional'])
@pytest.mark.parametrize('dims', [
    ('time', 'level', 'latitude', 'longitude'),
    ('time', 'level', 'longitude', 'latitude'),
    ('latitude', 'level', 'time', 'longitude'),
    ('longitude', 'time', 'latitude', 'level')], ids=lambda d: '-'.join(
        x[:3] for x in d))
def test_every_class_on_both_layouts_and_grids(grid, dims):
  from weatherbench2_b200 import derived_variables as dv, xarray_lite as xl
  lat, lon = dc.grid(grid)
  data = dc.fields(dc.shape_of(dims, lat, lon), 4)
  ds = dc.dataset(xl, dims, lat, lon, data)
  for kind in do.KINDS:
    got, fake = _run(dv.DERIVED_VARIABLE_DICT[kind].compute, ds)
    assert got.dims == dims and got.values.dtype == np.float32
    assert set(got.coords) == set(ds[dc.NAMES['u']].coords)
    want = do.compute(kind, dims, lat, lon, **data, level=np.array(
        (1000, 850, 500)))
    np.testing.assert_array_equal(got.values, _f32(want), err_msg=kind)
    call = fake.calls[-1]
    lon_contig = dims.index('latitude') < dims.index('longitude')
    assert call[6:] == ((lon.size, 1) if lon_contig else (1, lat.size))


@pytest.mark.parametrize('level', [(1000, 850, 700, 500, 250), (50, 250, 500),
                                   (500,)])
def test_vertical_velocity_levels_both_ways(level):
  from weatherbench2_b200 import derived_variables as dv, xarray_lite as xl
  dims = ('time', 'level', 'latitude', 'longitude')
  lat, lon = dc.grid('descending')
  data = dc.fields(dc.shape_of(dims, lat, lon, level), 6)
  ds = dc.dataset(xl, dims, lat, lon, data, level)
  got, _ = _run(dv.VerticalVelocity().compute, ds)
  want = do.compute('vertical_velocity', dims, lat, lon, **data,
                    level=np.array(level))
  np.testing.assert_array_equal(got.values, _f32(want))
  assert (got.values[:, 0] == 0).all()


def test_class_fields_match_the_reference():
  from weatherbench2_b200 import derived_variables as dv
  d = dv.DERIVED_VARIABLE_DICT
  uv = ['u_component_of_wind', 'v_component_of_wind']
  for name in ('divergence', 'vorticity', 'vertical_velocity'):
    assert d[name].base_variables == uv
  for name in ('geostrophic_wind_speed', 'u_component_of_geostrophic_wind',
               'v_component_of_geostrophic_wind'):
    assert d[name].base_variables == ['geopotential']
    assert d[name].core_dims == ((['longitude', 'latitude'],),
                                 ['longitude', 'latitude'])
  for name in ('ageostrophic_wind_speed', 'u_component_of_ageostrophic_wind',
               'v_component_of_ageostrophic_wind'):
    assert d[name].base_variables == uv + ['geopotential']
  assert d['vertical_velocity'].core_dims[1] == ['level', 'longitude',
                                                 'latitude']
  assert dv.WindVorticity(u_name='a', v_name='b').base_variables == ['a', 'b']
  assert dv.GeostrophicWindSpeed('zz').base_variables == ['zz']
  assert isinstance(d['vorticity'], dv._3DWindVariable)  # pylint: disable=protected-access


def test_errors():
  from weatherbench2_b200 import _lib, derived_variables as dv
  from weatherbench2_b200 import xarray_lite as xl
  lat, lon = dc.grid('descending')
  dims = ('time', 'level', 'latitude', 'longitude')
  data = dc.fields(dc.shape_of(dims, lat, lon), 1)
  ds = dc.dataset(xl, dims, lat, lon, {'u': data['u']})
  with pytest.raises(KeyError):
    _run(dv.WindDivergence().compute, ds)  # v missing
  with pytest.raises(KeyError):
    _run(dv.GeostrophicWindSpeed().compute, ds)
  # VerticalVelocity without a level dimension / coordinate
  d2 = ('time', 'latitude', 'longitude')
  flat = {k: a[:, 0] for k, a in data.items()}
  no_level = dc.dataset(xl, d2, lat, lon, flat)
  with pytest.raises(KeyError):
    _run(dv.VerticalVelocity().compute, no_level)
  scalar_level = xl.Dataset({dc.NAMES[k]: (d2, a) for k, a in flat.items()},
                            {'time': np.arange(2), 'latitude': lat,
                             'longitude': lon, 'level': ((), 500)})
  with pytest.raises((KeyError, ValueError)):
    _run(dv.VerticalVelocity().compute, scalar_level)
  # fewer than 2 points along an axis (np.gradient's edge_order + 1)
  for la, lo in ((lat[:1], lon), (lat, lon[:1])):
    small = dc.dataset(xl, dims, la, lo, {
        k: np.zeros(dc.shape_of(dims, la, lo), np.float32) for k in 'uvz'})
    with pytest.raises((ValueError, _lib.Wb2Error)):
      _run(dv.WindVorticity().compute, small)
  # two points are enough
  two = dc.dataset(xl, dims, lat[:2], lon[:2], {
      k: data[k][:, :, :2, :2].copy() for k in 'uvz'})
  got, _ = _run(dv.WindVorticity().compute, two)
  assert got.shape == (2, 3, 2, 2)


def test_every_class_in_the_metric_loop():
  from oracle import wb2_oracle as orc
  from weatherbench2_b200 import config, derived_variables as dv, evaluation
  from weatherbench2_b200 import metrics, regions, xarray_lite as xl
  dims = ('time', 'level', 'latitude', 'longitude')
  lat, lon = dc.grid('nonuniform32')
  shape = dc.shape_of(dims, lat, lon, ntime=3)
  f, t = dc.fields(shape, 7, nan=False), dc.fields(shape, 8, nan=False)
  fds = dc.dataset(xl, dims, lat, lon, f, ntime=3)
  tds = dc.dataset(xl, dims, lat, lon, t, ntime=3)
  ec = config.Eval(metrics={'mse': metrics.MSE()},
                   regions={'extra_tropics': regions.ExtraTropicalRegion()},
                   derived_variables={k: dv.DERIVED_VARIABLE_DICT[k]
                                      for k in do.KINDS})
  res, _ = _run(evaluation._metric_and_region_loop, fds, tds, ec,  # pylint: disable=protected-access
                skipna=False)
  for kind in do.KINDS:
    fs = _f32(do.compute(kind, dims, lat, lon, **f, level=np.array(
        (1000, 850, 500))))
    ts = _f32(do.compute(kind, dims, lat, lon, **t, level=np.array(
        (1000, 850, 500))))
    with np.errstate(invalid='ignore'):
      want, wd = orc.mse(fs, dims, ts, dims, lat, lon,
                         region=orc.ExtraTropicalRegion())
      want, wd = orc.time_mean(want, wd, avg_dim='time')
    got = res[kind].isel(metric=0, region=0)
    a, b, _ = orc.align(np.asarray(got.values), got.dims, want, wd)
    assert np.isfinite(a).all(), kind
    np.testing.assert_allclose(a, b, rtol=1e-5, err_msg=kind)


def test_by_init_evaluation_with_vorticity(tmp_path):
  """evaluate_in_memory, by init, with `vorticity` derived on forecast and
  (gathered) truth."""
  from oracle import wb2_oracle as orc
  from weatherbench2_b200 import config, derived_variables as dv, evaluation
  from weatherbench2_b200 import metrics, xarray_lite as xl
  lat, lon = _grid(19, 36)
  level = np.array([500, 850])
  init = np.arange('2020-01-01T00', '2020-01-03T00', 12,
                   dtype='datetime64[h]').astype('datetime64[ns]')
  lead = np.arange(0, 36, 12).astype('timedelta64[h]').astype(
      'timedelta64[ns]')
  times = np.arange('2019-12-31T00', '2020-01-05T00', 12,
                    dtype='datetime64[h]').astype('datetime64[ns]')
  fd = ('time', 'prediction_timedelta', 'level', 'latitude', 'longitude')
  td = ('time', 'level', 'latitude', 'longitude')
  rs = np.random.RandomState(3)
  fshape = (init.size, lead.size, level.size, lat.size, lon.size)
  tshape = (times.size, level.size, lat.size, lon.size)
  fu, fv = (rs.normal(scale=10, size=fshape).astype(np.float32)
            for _ in range(2))
  tu, tv = (rs.normal(scale=10, size=tshape).astype(np.float32)
            for _ in range(2))
  names = ('u_component_of_wind', 'v_component_of_wind')
  forecast = xl.Dataset({names[0]: (fd, fu), names[1]: (fd, fv)},
                        {'time': init, 'prediction_timedelta': lead,
                         'level': level, 'latitude': lat, 'longitude': lon})
  truth = xl.Dataset({names[0]: (td, tu), names[1]: (td, tv)},
                     {'time': times, 'level': level, 'latitude': lat,
                      'longitude': lon})
  paths = config.Paths(forecast=forecast, obs=truth,
                       output_dir=str(tmp_path))
  sel = config.Selection(variables=['vorticity'], levels=[500, 850],
                         time_slice=slice(init[0], init[-1]))
  data_config = config.Data(selection=sel, paths=paths, by_init=True)
  ec = config.Eval(metrics={'mse': metrics.MSE()},
                   derived_variables={'vorticity': dv.WindVorticity()})
  res, fake = _run(evaluation.evaluate_in_memory, data_config, {'deterministic': ec})
  assert any(c[0] == 'wind_dynamics' for c in fake.calls)
  got = res['deterministic']['vorticity']
  # truth at valid time init + lead
  idx = np.searchsorted(times, init[:, None] + lead[None, :])
  tvort = do.compute('vorticity', td, lat, lon, u=tu, v=tv)[idx]
  fvort = do.compute('vorticity', fd, lat, lon, u=fu, v=fv)
  want, wd = orc.mse(_f32(fvort), fd, _f32(tvort), fd, lat, lon)
  want, wd = orc.time_mean(want, wd, avg_dim='time')
  wd = tuple('lead_time' if d == 'prediction_timedelta' else d for d in wd)
  g = got.isel(metric=0) if 'metric' in got.dims else got
  a, b, _ = orc.align(np.asarray(g.values), g.dims, want, wd)
  np.testing.assert_allclose(a, b, rtol=1e-5)

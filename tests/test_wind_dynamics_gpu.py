"""GPU tests of wb2_wind_dynamics (csrc/wind_dynamics.cu) and the derived
variables built on it (weatherbench2/derived_variables.py:102-338): every kind
bit-equal to the float64 oracle (tests/dynamics_oracle.py) rounded to float32
on a 0.25-degree uniform grid and a 32 x 64 non-uniform one, in both field
layouts, with NaN cells, the pole rows and the equator row; torch CUDA and
NumPy inputs; float64 inputs within the documented bound; every argument
error of the entry; and the variables inside an evaluation."""
import numpy as np
import pytest

import dynamics_cases as dc
import dynamics_oracle as do
from oracle import wb2_oracle as orc

pytestmark = pytest.mark.gpu

LAYOUTS = {'lat_lon': ('time', 'level', 'latitude', 'longitude'),
           'lon_lat': ('time', 'level', 'longitude', 'latitude')}


def _assert_bit_equal(got, want64, what):
  want = np.asarray(want64).astype(np.float32)
  got = np.asarray(got)
  assert got.dtype == np.float32, what
  np.testing.assert_array_equal(np.isnan(got), np.isnan(want), err_msg=what)
  same = (got.view(np.uint32) == want.view(np.uint32)) | np.isnan(want)
  if not same.all():
    i = np.argwhere(~same)[0]
    raise AssertionError(f'{what}: {(~same).sum()} cells differ, first at '
                         f'{tuple(i)}: {got[tuple(i)]!r} vs {want[tuple(i)]!r}')


def _expected(kind, dims, lat, lon, data, level=(1000, 850, 500)):
  return do.compute(kind, dims, lat, lon, **data, level=np.asarray(level))


@pytest.mark.parametrize('layout', sorted(LAYOUTS))
@pytest.mark.parametrize('grid', ['uniform721', 'nonuniform32'])
def test_every_kind_is_bit_equal_to_the_oracle(grid, layout):
  import torch
  from weatherbench2_b200 import derived_variables as dv, xarray_lite as xl
  dims = LAYOUTS[layout]
  lat, lon = dc.grid(grid)
  level = (1000, 850, 500) if grid == 'nonuniform32' else (850, 500)
  shape = dc.shape_of(dims, lat, lon, level)
  data = dc.fields(shape, 11)
  ilat = dims.index('latitude')
  eq = int(np.argmin(np.abs(lat)))
  assert lat[eq] == 0 and abs(lat[0]) == 90 and abs(lat[-1]) == 90
  # a row of z constant along longitude on the equator: 0 / 0 = NaN there
  sl = [slice(None)] * len(dims)
  sl[ilat] = eq
  sl[0] = 0
  data['z'][tuple(sl)] = 5e4
  host = dc.dataset(xl, dims, lat, lon, data, level)
  dev = dc.dataset(xl, dims, lat, lon, data, level,
                   wrap=lambda a: torch.from_numpy(a).cuda())
  for kind in do.KINDS:
    want = _expected(kind, dims, lat, lon, data, level)
    var = dv.DERIVED_VARIABLE_DICT[kind]
    got = var.compute(host)
    assert got.dims == dims and isinstance(got.values, np.ndarray)
    _assert_bit_equal(got.values, want, f'{kind} numpy')
    gd = var.compute(dev)
    assert gd.dims == dims and gd.data.is_cuda
    _assert_bit_equal(gd.data.cpu().numpy(), want, f'{kind} cuda')
    if 'geostrophic' in kind:
      w = np.moveaxis(np.asarray(want), ilat, 0)
      assert not np.isfinite(w[eq]).all(), kind  # inf / NaN on the equator
      if kind == 'v_component_of_geostrophic_wind':
        assert (w[0] == 0).all() and (w[-1] == 0).all()  # poles zeroed


def test_nan_cells_and_their_neighbours():
  """A NaN spreads to its stencil neighbours exactly as np.gradient spreads
  it, and nowhere else; pole rows of _d_dx stay 0 even where the input is
  NaN."""
  from weatherbench2_b200 import derived_variables as dv, xarray_lite as xl
  dims = ('latitude', 'longitude')
  lat, lon = dc.grid('nonuniform32')
  data = dc.fields((lat.size, lon.size), 5, nan=False)
  data['u'][0, 10] = np.nan      # on the south pole row
  data['u'][15, 0] = np.nan      # equator, longitude edge
  data['v'][31, 63] = np.nan     # corner
  data['v'][9, 30] = np.nan
  data['z'][20, 20] = np.nan
  ds = dc.dataset(xl, dims, lat, lon, data)
  for kind in ('divergence', 'vorticity', 'geostrophic_wind_speed',
               'ageostrophic_wind_speed'):
    got = dv.DERIVED_VARIABLE_DICT[kind].compute(ds).values
    want = _expected(kind, dims, lat, lon, data)
    _assert_bit_equal(got, want, kind)
  div = dv.WindDivergence().compute(ds).values
  assert np.isfinite(div[0, 9:12]).all()  # pole row: _d_dx(u) is 0, not NaN


def test_vertical_velocity_with_levels_descending_and_ascending():
  import torch
  from weatherbench2_b200 import derived_variables as dv, xarray_lite as xl
  lat, lon = dc.grid('uniform721')
  for level in ((1000, 925, 850, 700, 600, 500, 400, 300, 250, 200, 150, 100,
                 50), (50, 300, 500, 850)):
    dims = ('time', 'level', 'latitude', 'longitude')
    data = dc.fields(dc.shape_of(dims, lat, lon, level, ntime=1), 3)
    data.pop('z')
    ds = dc.dataset(xl, dims, lat, lon, data, level, ntime=1,
                    wrap=lambda a: torch.from_numpy(a).cuda())
    got = dv.VerticalVelocity().compute(ds)
    want = _expected('vertical_velocity', dims, lat, lon, data, level)
    _assert_bit_equal(got.data.cpu().numpy(), want, str(level))
    assert (got.data[:, 0] == 0).all()


def _abs_gradient(a, coord, axis):
  """sum |coefficient * f| of np.gradient's stencil at every index."""
  a = np.moveaxis(np.abs(np.asarray(a, np.float64)), axis, -1)
  x = np.asarray(coord, np.float64)
  dx = np.diff(x)
  out = np.empty(a.shape)
  out[..., 0] = (a[..., 1] + a[..., 0]) / abs(dx[0])
  out[..., -1] = (a[..., -1] + a[..., -2]) / abs(dx[-1])
  d1, d2 = dx[:-1], dx[1:]
  ca = np.abs(-d2 / (d1 * (d1 + d2)))
  cb = np.abs((d2 - d1) / (d1 * d2))
  cc = np.abs(d1 / (d2 * (d1 + d2)))
  out[..., 1:-1] = ca * a[..., :-2] + cb * a[..., 1:-1] + cc * a[..., 2:]
  return np.moveaxis(out, -1, axis)


def _float64_bound(kind, dims, lat, lon, data, level):
  """Bound of |float64-input result - reference float64 arithmetic| per cell
  (DESIGN.md, "Wind dynamics"): 2^-22 times the stencil magnitude, scaled as
  the output, plus 2^-23 of the output."""
  ilat, ilon = dims.index('latitude'), dims.index('longitude')
  cos = np.cos(np.deg2rad(do._along(lat, dims, 'latitude')))  # pylint: disable=protected-access
  f = np.abs(2 * do.OMEGA * np.sin(np.deg2rad(do._along(lat, dims, 'latitude'))))  # pylint: disable=protected-access
  m = do.METERS_PER_DEGREE

  def sx(a):
    with np.errstate(divide='ignore', invalid='ignore'):
      return np.where(cos > 1e-6, _abs_gradient(a, lon, ilon) / cos / m, 0)

  def sy(a):
    return _abs_gradient(a, lat, ilat) / m

  with np.errstate(divide='ignore', invalid='ignore'):
    b = {'divergence': lambda: sx(data['u']) + sy(data['v']),
         'vorticity': lambda: sx(data['v']) + sy(data['u']),
         'u_component_of_geostrophic_wind': lambda: sy(data['z']) / f,
         'v_component_of_geostrophic_wind': lambda: sx(data['z']) / f,
         'geostrophic_wind_speed': lambda: (sy(data['z']) + sx(data['z'])) / f,
         'u_component_of_ageostrophic_wind':
             lambda: np.abs(data['u']) + sy(data['z']) / f,
         'v_component_of_ageostrophic_wind':
             lambda: np.abs(data['v']) + sx(data['z']) / f,
         'ageostrophic_wind_speed':
             lambda: (np.abs(data['u']) + np.abs(data['v']) +
                      (sy(data['z']) + sx(data['z'])) / f)}
    if kind == 'vertical_velocity':
      bd = np.moveaxis(sx(data['u']) + sy(data['v']), dims.index('level'), 0)
      dp = np.abs(np.diff(100 * np.asarray(level, np.float64)))
      steps = dp[:, None, None, None] * (bd[1:] + bd[:-1]) / 2
      out = np.concatenate([np.zeros_like(bd[:1]), np.cumsum(steps, axis=0)])
      return np.moveaxis(out, 0, dims.index('level'))
    return b[kind]()


def test_float64_input_within_the_documented_bound():
  from weatherbench2_b200 import derived_variables as dv, xarray_lite as xl
  dims = LAYOUTS['lat_lon']
  lat, lon = dc.grid('nonuniform32')
  level = (1000, 850, 500)
  rs = np.random.RandomState(2)
  shape = dc.shape_of(dims, lat, lon, level)
  data = {'u': rs.normal(scale=10, size=shape),
          'v': rs.normal(scale=10, size=shape),
          'z': 5e4 + rs.normal(scale=300, size=shape)}
  ds = dc.dataset(xl, dims, lat, lon, data, level)
  for kind in do.KINDS:
    got = dv.DERIVED_VARIABLE_DICT[kind].compute(ds).values
    assert got.dtype == np.float32
    want = _expected(kind, dims, lat, lon, data, level)  # float64 throughout
    fin = np.isfinite(want)
    np.testing.assert_array_equal(np.isfinite(got), fin, err_msg=kind)
    bound = (2.0**-22 * _float64_bound(kind, dims, lat, lon, data, level) +
             2.0**-23 * np.abs(want))
    err = np.abs(got.astype(np.float64) - want)
    assert (err[fin] <= bound[fin]).all(), (kind, (err[fin] / bound[fin]).max())
    # and it is exactly the float32 result of the data rounded to float32
    d32 = {k: a.astype(np.float32) for k, a in data.items()}
    got32 = dv.DERIVED_VARIABLE_DICT[kind].compute(
        dc.dataset(xl, dims, lat, lon, d32, level)).values
    np.testing.assert_array_equal(got, got32, err_msg=kind)


def test_every_argument_error_is_reported():
  from weatherbench2_b200 import _lib, _derived_wind as dw
  ctx = _lib.default_context()
  lat, lon = dc.grid('nonuniform32')
  lt, lu = dw.gradient_table(lat)
  ot, ou = dw.gradient_table(lon)
  cos = np.cos(np.deg2rad(lat))
  cor = dw.coriolis_parameter(lat)
  pres = np.array([1e5, 5e4])
  n = 2 * lat.size * lon.size
  bufs = [ctx.malloc(4 * n) for _ in range(4)]
  u, v, z, out = bufs
  good = dict(kind=0, u=u, v=v, z=z, nouter=1, nlev=2, nlat=lat.size,
              nlon=lon.size, lat_stride=lon.size, lon_stride=1, lat_coef=lt,
              lat_uniform=lu, lon_coef=ot, lon_uniform=ou, cos_lat=cos,
              coriolis=cor, pressure=pres, out=out)
  try:
    before = ctx.launch_count
    for kind in range(9):
      ctx.wind_dynamics(**dict(good, kind=kind))
    ctx.wind_dynamics(**dict(good, lat_stride=1, lon_stride=lat.size))
    ctx.synchronize()
    assert ctx.launch_count - before == 10  # one launch per call
    bad = [dict(kind=-1), dict(kind=9), dict(nouter=-1), dict(nlev=-1),
           dict(nlat=1, lat_coef=lt[:1], cos_lat=cos[:1], coriolis=cor[:1],
                lat_stride=lon.size),
           dict(nlon=1, lon_coef=ot[:1], lat_stride=1),
           dict(lat_stride=lon.size + 1), dict(lon_stride=2),
           dict(lat_stride=1, lon_stride=1), dict(out=None),
           dict(u=None), dict(v=None), dict(kind=1, u=None),
           dict(kind=2, pressure=None), dict(kind=3, z=None),
           dict(kind=4, coriolis=None), dict(kind=7, u=None),
           dict(kind=8, v=None), dict(kind=6, z=None),
           dict(lat_coef=None), dict(lon_coef=None), dict(cos_lat=None)]
    for change in bad:
      with pytest.raises(_lib.Wb2Error):
        ctx.wind_dynamics(**dict(good, **change))
    # the operand a kind does not read may be NULL
    ctx.wind_dynamics(**dict(good, kind=7, v=None))
    ctx.wind_dynamics(**dict(good, kind=8, u=None))
    ctx.wind_dynamics(**dict(good, kind=3, u=None, v=None, pressure=None))
    ctx.wind_dynamics(**dict(good, kind=0, z=None, coriolis=None))
    ctx.wind_dynamics(**dict(good, nouter=0))
    ctx.synchronize()
  finally:
    for p in bufs:
      ctx.free(p)


def _eval(fds, tds, names, regions=None):
  from weatherbench2_b200 import config, derived_variables as dv, evaluation
  from weatherbench2_b200 import metrics
  ec = config.Eval(metrics={'mse': metrics.MSE()}, regions=regions,
                   derived_variables={n: dv.DERIVED_VARIABLE_DICT[n]
                                      for n in names})
  return evaluation._metric_and_region_loop(fds, tds, ec, skipna=False)  # pylint: disable=protected-access


def test_geostrophic_wind_speed_in_an_evaluation():
  """Finite over an ExtraTropicalRegion; over the globe non-finite exactly
  where the oracle's metric is."""
  from weatherbench2_b200 import regions, xarray_lite as xl
  dims = ('time', 'latitude', 'longitude')
  lat, lon = dc.grid('nonuniform32')
  shape = dc.shape_of(dims, lat, lon, ntime=3)
  f = dc.fields(shape, 21, nan=False)
  t = dc.fields(shape, 22, nan=False)
  # time 1: z constant on the equator in both -> 0/0 = NaN there
  for d in (f, t):
    d['z'][1, int(np.argmin(np.abs(lat)))] = 5e4
  fds = dc.dataset(xl, dims, lat, lon, {'z': f['z']}, ntime=3)
  tds = dc.dataset(xl, dims, lat, lon, {'z': t['z']}, ntime=3)
  res = _eval(fds, tds, ['geostrophic_wind_speed'],
              {'global': regions.SliceRegion(),
               'extra_tropics': regions.ExtraTropicalRegion()})
  got = res['geostrophic_wind_speed']
  gv = np.asarray(got.values)
  ri = got.dims.index('region')
  names = list(np.asarray(got.coords['region'].values))
  assert np.isfinite(np.take(gv, names.index('extra_tropics'), axis=ri)).all()
  fs = do.compute('geostrophic_wind_speed', dims, lat, lon, z=f['z'])
  ts = do.compute('geostrophic_wind_speed', dims, lat, lon, z=t['z'])
  with np.errstate(invalid='ignore'):
    want, wd = orc.mse(fs.astype(np.float32), dims, ts.astype(np.float32),
                       dims, lat, lon)
    want, wd = orc.time_mean(want, wd, avg_dim='time')
  glob = np.take(gv, names.index('global'), axis=ri)
  np.testing.assert_array_equal(np.isfinite(glob).reshape(-1),
                                np.isfinite(want).reshape(-1))


def test_vorticity_from_cuda_tensors_in_an_evaluation():
  import torch
  from weatherbench2_b200 import xarray_lite as xl
  dims = ('time', 'level', 'latitude', 'longitude')
  lat, lon = dc.grid('uniform721')
  shape = dc.shape_of(dims, lat, lon, (850, 500))
  f = dc.fields(shape, 31, nan=False)
  t = dc.fields(shape, 32, nan=False)
  cuda = lambda a: torch.from_numpy(a).cuda()  # noqa: E731
  fds = dc.dataset(xl, dims, lat, lon, {k: f[k] for k in 'uv'}, (850, 500),
                   wrap=cuda)
  tds = dc.dataset(xl, dims, lat, lon, {k: t[k] for k in 'uv'}, (850, 500),
                   wrap=cuda)
  res = _eval(fds, tds, ['vorticity'])
  got = res['vorticity'].isel(metric=0)
  fs = do.compute('vorticity', dims, lat, lon, u=f['u'], v=f['v'])
  ts = do.compute('vorticity', dims, lat, lon, u=t['u'], v=t['v'])
  want, wd = orc.mse(fs.astype(np.float32), dims, ts.astype(np.float32), dims,
                     lat, lon)
  want, wd = orc.time_mean(want, wd, avg_dim='time')
  a, b, _ = orc.align(np.asarray(got.values), got.dims, want, wd)
  np.testing.assert_allclose(a, b, rtol=1e-5)

"""GPU: wb2_column_integral through the column-integral classes, against
tests/column_oracle.py.  Total column and IVT are bit-equal to the oracle, NaN
positions included, for CUDA and NumPy input; EKE for float32 data is within
one float32 ulp (the zonal sum of float32 values in float64 is exact for
these fields, whatever its order).  The cases fail for the sum taken as
sum_k c_k y_k instead of the pair form, a float32 accumulation, a dropped last
level pair, an IVT window one level off, and a zonal mean that counts NaN
cells."""
import numpy as np
import pytest

import column_oracle as co

pytestmark = pytest.mark.gpu

Q, U, V = 'specific_humidity', 'u_component_of_wind', 'v_component_of_wind'
TLLL = ('time', 'level', 'latitude', 'longitude')
LEVELS13 = (50, 100, 150, 200, 250, 300, 400, 500, 600, 700, 850, 925, 1000)
LEVELS37 = (1, 2, 3, 5, 7, 10, 20, 30, 50, 70, 100, 125, 150, 175, 200, 225,
            250, 300, 350, 400, 450, 500, 550, 600, 650, 700, 750, 775, 800,
            825, 850, 875, 900, 925, 950, 975, 1000)


def _fields(shape, seed, dtype=np.float32, dims=TLLL):
  rs = np.random.RandomState(seed)
  q = np.abs(rs.normal(scale=4e-3, size=shape)).astype(dtype)
  u = (5 + rs.normal(scale=12, size=shape)).astype(dtype)
  v = rs.normal(scale=8, size=shape).astype(dtype)
  q.reshape(-1)[5] = np.nan

  def at(lat, lon):
    i = [0] * len(shape)
    i[dims.index('latitude')], i[dims.index('longitude')] = lat, lon
    return tuple(i)

  # one zonal row of v that is NaN throughout (latitude 1), and a NaN u cell in
  # another row (latitude 2), so that a zonal mean that counts NaN cells shows
  # in every layout
  v[at(1, slice(None))] = np.nan
  u[at(2, 3)] = np.nan
  return {Q: q, U: u, V: v}


def _dataset(dims, fields, level, lat, lon, device):
  import torch
  from weatherbench2_b200 import xarray_lite as xl
  coords = {'time': np.arange(fields[Q].shape[dims.index('time')])
            if 'time' in dims else None, 'level': np.asarray(level),
            'latitude': lat, 'longitude': lon}
  wrap = (lambda a: torch.from_numpy(a).cuda()) if device else (lambda a: a)
  return xl.Dataset({k: (dims, wrap(a)) for k, a in fields.items()},
                    {k: c for k, c in coords.items() if k in dims})


def _bits(got, want, what):
  got = got.detach().cpu().numpy() if hasattr(got, 'detach') else got
  assert got.dtype == want.dtype, what
  np.testing.assert_array_equal(np.isnan(got), np.isnan(want), err_msg=what)
  np.testing.assert_array_equal(got, want, err_msg=what)


def _ulp(got, want, what):
  got = got.detach().cpu().numpy() if hasattr(got, 'detach') else got
  np.testing.assert_array_equal(np.isnan(got), np.isnan(want), err_msg=what)
  ok = np.isnan(want) | (np.abs(got - want) <= np.spacing(np.abs(want)))
  assert ok.all(), what


def _check_all(dims, level, lat, lon, dtype, seed, device, windows=((300, 1000),)):
  from weatherbench2_b200 import derived_variables as dv
  shape = tuple({'time': 2, 'level': len(level), 'latitude': lat.size,
                 'longitude': lon.size}[d] for d in dims)
  f = _fields(shape, seed, dtype, dims)
  ds = _dataset(dims, f, level, lat, lon, device)
  la, lo = dims.index('level'), dims.index('longitude')
  tc = dv.DERIVED_VARIABLE_DICT['total_column_vapor'].compute(ds)
  assert tc.dims == tuple(d for d in dims if d != 'level')
  assert (getattr(tc.data, 'is_cuda', False)) == device
  _bits(tc.data, co.rounded(co.total_column(f[Q], level, la), dtype), 'tc')
  for lmin, lmax in windows:
    ivt = dv.IntegratedWaterTransport(level_min=lmin,
                                      level_max=lmax).compute(ds)
    want = co.ivt(f[Q], f[U], f[V], level, la, lmin, lmax)
    _bits(ivt.data, co.rounded(want, dtype), f'ivt {lmin}..{lmax}')
  eke = dv.DERIVED_VARIABLE_DICT['eddy_kinetic_energy'].compute(ds)
  want = co.rounded(co.eke(f[U], f[V], level, la, lo), dtype)
  if dtype == np.float32:
    _ulp(eke.data, want, 'eke')
  else:
    got = eke.values
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
    np.testing.assert_allclose(got, want, rtol=1e-13)
  return f


@pytest.mark.parametrize('device', [True, False], ids=['cuda', 'numpy'])
@pytest.mark.parametrize('level', [LEVELS13, LEVELS37], ids=['13', '37'])
@pytest.mark.parametrize('dims', [TLLL, ('time', 'level', 'longitude',
                                         'latitude')], ids=['latlon', 'lonlat'])
def test_721x1440(dims, level, device):
  lat, lon = np.linspace(-90, 90, 721), np.arange(1440) * 0.25
  _check_all(dims, level, lat, lon, np.float32, 1, device)


@pytest.mark.parametrize('device', [True, False], ids=['cuda', 'numpy'])
@pytest.mark.parametrize('dtype', [np.float32, np.float64])
@pytest.mark.parametrize('dims', [
    TLLL, ('time', 'level', 'longitude', 'latitude'),
    ('level', 'latitude', 'time', 'longitude'),
    ('time', 'latitude', 'longitude', 'level')],
                         ids=lambda d: '-'.join(x[:3] for x in d))
def test_small_nonuniform_grid(dims, dtype, device):
  # 33 rows: the (longitude, latitude) kernel's last tile of 8 rows is partial
  lat = np.sort(np.r_[np.linspace(-90, 90, 31), 3.0, 7.5])
  lon = np.linspace(0, 355, 72)
  level = (70, 137.5, 300, 312.25, 500, 700, 850, 1000)
  _check_all(dims, level, lat, lon, dtype, 2, device,
             windows=((300, 1000), (None, None), (312.25, 850), (301, 999),
                      (1000, 300)))


@pytest.mark.parametrize('device', [True, False], ids=['cuda', 'numpy'])
def test_one_level_and_the_empty_window(device):
  from weatherbench2_b200 import derived_variables as dv
  lat, lon = np.linspace(-90, 90, 9), np.arange(16) * 22.5
  for level in ((500,), (1000, 850, 500)):
    f = _fields((2, len(level), 9, 16), 3)
    ds = _dataset(TLLL, f, level, lat, lon, device)
    if len(level) == 1:
      for var in (dv.TotalColumnWater(), dv.EddyKineticEnergy(),
                  dv.IntegratedWaterTransport()):
        assert (var.compute(ds).values == 0).all()
    else:  # descending levels: pandas' slice is empty, the reference gives 0
      assert (dv.IntegratedWaterTransport().compute(ds).values == 0).all()
      tc = dv.TotalColumnWater().compute(ds).values
      _bits(tc, co.rounded(co.total_column(f[Q], level, 1), np.float32),
            'descending tc')


def test_every_argument_error_and_one_launch_per_call():
  import torch
  from weatherbench2_b200 import _lib
  ctx = _lib.default_context()
  x = torch.zeros((2, 5, 6, 8), device='cuda')
  out = torch.empty((2, 6, 8), device='cuda')
  w = np.full(4, 50.0)
  good = dict(kind=1, dtype=_lib.F32, q=x.data_ptr(), u=x.data_ptr(),
              v=x.data_ptr(), nouter=2, outer_stride=5 * 48, nlev=5, ninner=48,
              nlon=8, lon_stride=1, weight=w, out=out.data_ptr())
  bad = [dict(kind=3), dict(kind=-1), dict(dtype=2), dict(nouter=-1),
         dict(nlev=-1), dict(ninner=-1), dict(outer_stride=5 * 48 - 1),
         dict(q=None), dict(u=None), dict(v=None), dict(out=None),
         dict(weight=None),
         dict(kind=0, q=None), dict(kind=2, u=None), dict(kind=2, v=None),
         dict(kind=2, nlon=0), dict(kind=2, nlon=7), dict(kind=2, lon_stride=8),
         dict(kind=2, lon_stride=0), dict(kind=2, nlon=48, lon_stride=2),
         dict(kind=2, nlon=1 << 20, ninner=1 << 20, outer_stride=5 << 20),
         dict(kind=2, nlon=1 << 17, ninner=1 << 18, outer_stride=5 << 18,
              lon_stride=2)]
  for change in bad:
    with pytest.raises(_lib.Wb2Error):
      ctx.column_integral(**dict(good, **change))
  ctx.synchronize()
  before = ctx.launch_count
  ctx.column_integral(**good)
  ctx.column_integral(**dict(good, kind=0, u=None, v=None))
  ctx.column_integral(**dict(good, kind=2, q=None))
  ctx.column_integral(**dict(good, kind=2, q=None, lon_stride=6))
  ctx.column_integral(**dict(good, nlev=1, weight=None))
  ctx.column_integral(**dict(good, nlev=0, weight=None))
  ctx.synchronize()
  assert ctx.launch_count - before == 6
  assert (out == 0).all()
  ctx.column_integral(**dict(good, nouter=0))  # nothing to do
  ctx.column_integral(**dict(good, ninner=0, outer_stride=0))
  ctx.synchronize()
  assert ctx.launch_count - before == 6


def test_one_launch_per_variable():
  from weatherbench2_b200 import _lib, derived_variables as dv
  ctx = _lib.default_context()
  lat, lon = np.linspace(-90, 90, 9), np.arange(16) * 22.5
  ds = _dataset(TLLL, _fields((2, 4, 9, 16), 4), (300, 500, 850, 1000), lat,
                lon, True)
  for name in ('total_column_vapor', 'integrated_vapor_transport',
               'eddy_kinetic_energy'):
    before = ctx.launch_count
    dv.DERIVED_VARIABLE_DICT[name].compute(ds)
    ctx.synchronize()
    assert ctx.launch_count - before == 1, name


@pytest.mark.parametrize('device', [True, False], ids=['cuda', 'numpy'])
def test_ivt_and_eke_inside_an_evaluation(device):
  """MSE over the derived IVT and EKE on the device equals the same loop fed
  the oracle's values as plain variables."""
  import torch
  from weatherbench2_b200 import config, derived_variables as dv, evaluation
  from weatherbench2_b200 import metrics, regions, xarray_lite as xl
  lat, lon = np.linspace(-90, 90, 33), np.arange(64) * 5.625
  level = LEVELS13
  shape = (3, 13, 33, 64)
  f, t = _fields(shape, 5), _fields(shape, 6)
  for x in (f, t):  # the metric sees finite fields
    for a in x.values():
      np.nan_to_num(a, copy=False, nan=1e-3)
  fds = _dataset(TLLL, f, level, lat, lon, device)
  tds = _dataset(TLLL, t, level, lat, lon, device)
  names = ('integrated_vapor_transport', 'eddy_kinetic_energy')
  ms = {'mse': metrics.MSE()}
  rg = {'global': regions.SliceRegion(),
        'extra_tropics': regions.ExtraTropicalRegion()}
  ec = config.Eval(metrics=ms, regions=rg, derived_variables={
      k: dv.DERIVED_VARIABLE_DICT[k] for k in names})
  res = evaluation._metric_and_region_loop(fds, tds, ec, skipna=False)  # pylint: disable=protected-access
  d2 = ('time', 'latitude', 'longitude')
  wrap = (lambda a: torch.from_numpy(a).cuda()) if device else (lambda a: a)

  def plain(x):
    return xl.Dataset(
        {'integrated_vapor_transport': (d2, wrap(co.rounded(
            co.ivt(x[Q], x[U], x[V], level, 1), np.float32))),
         'eddy_kinetic_energy': (d2, wrap(co.rounded(
             co.eke(x[U], x[V], level, 1, 3), np.float32)))},
        {'time': np.arange(3), 'latitude': lat, 'longitude': lon})

  want = evaluation._metric_and_region_loop(plain(f), plain(t),  # pylint: disable=protected-access
                                            config.Eval(metrics=ms, regions=rg),
                                            skipna=False)
  for k in names:
    a, b = np.asarray(res[k].values), np.asarray(want[k].values)
    assert np.isfinite(a).all(), k
    np.testing.assert_allclose(a, b, rtol=1e-6, err_msg=k)

"""The *_host entries (csrc/host_stream.cu): double-buffered streaming of host
slabs, the LRU slab cache for truth / climatology, the transfer accounting, and
the operators that use them for NumPy inputs.  Every result is compared with
the device-resident entry of the same kernel (bit-identical: same kernels, same
order) and, where cheap, with the oracle."""
import numpy as np
import pytest

from oracle import wb2_oracle as orc

pytestmark = pytest.mark.gpu


@pytest.fixture
def small_stage_ctx(monkeypatch):
  """A private context whose staging buffers hold only a few slabs, so that the
  group loop, the double buffering and the cache eviction paths all run."""
  from weatherbench2_b200 import _lib
  monkeypatch.setenv('WB2_STAGE_MB', '1')
  ctx = _lib.Context(0)
  yield ctx
  ctx.close()


def _np(v):
  return v.cpu().numpy() if hasattr(v, 'cpu') else np.asarray(v)


def _weights(ctx, nlat, nlon, regions=(None,)):
  from weatherbench2_b200 import _spatial as sp
  lat = np.linspace(-90, 90, nlat)
  lon = np.linspace(0, 360, nlon, endpoint=False)
  (_, spec), = sp.build_weights(ctx, lat, lon, list(regions), 'lat_lon', nlon)
  return lat, lon, spec


def _det_device(ctx, f, t, c, off_f, off_t, off_c, spec, skipna):
  """Reference result: the same operands uploaded whole, device entry."""
  from weatherbench2_b200 import _lib
  df, dt_, dc = ctx.to_device(f), ctx.to_device(t), ctx.to_device(c)
  base = min(df, dt_, dc)
  n = off_f.size
  out = ctx.malloc(n * _lib.DET_NSTAT * 8)
  try:
    ctx.det_metrics(base, base, base, _lib.F32, off_f + (df - base) // 4,
                    off_t + (dt_ - base) // 4, off_c + (dc - base) // 4, spec,
                    skipna, out)
    return ctx.from_device(out, (n, 1, _lib.DET_NSTAT), np.float64)
  finally:
    for p in (df, dt_, dc, out):
      ctx.free(p)


@pytest.mark.parametrize('cache_slabs', [0, 7, 1000])
def test_det_host_chunk_sweep_with_slab_cache(small_stage_ctx, cache_slabs):
  """A sweep over init times like evaluation.py:583-599: chunk i needs truth /
  climatology slabs of valid times i .. i + nlead - 1, so consecutive chunks
  share all but one.  cache_slabs = 7 is smaller than a chunk's working set
  (eviction inside a call), 1000 holds everything."""
  from weatherbench2_b200 import _lib
  ctx = small_stage_ctx
  nlat, nlon, nlead, nlev, ninit = 33, 64, 4, 3, 5
  slab = nlat * nlon
  _, _, spec = _weights(ctx, nlat, nlon)
  rs = np.random.RandomState(0)
  ntime = ninit + nlead
  truth = rs.standard_normal((ntime, nlev, nlat, nlon)).astype(np.float32)
  clim = rs.standard_normal((ntime, nlev, nlat, nlon)).astype(np.float32)
  slab_bytes = (slab + 63) // 64 * 64 * 4
  ctx.set_slab_cache(cache_slabs * slab_bytes)
  ctx.reset_transfer_stats()
  h2d = []
  try:
    for i in range(ninit):
      f = rs.standard_normal((nlead, nlev, nlat, nlon)).astype(np.float32)
      if i == 2:
        f[1, 0, 3, 5] = np.nan
      off_f = np.arange(nlead * nlev, dtype=np.int64) * slab
      lead_t = (i + np.arange(nlead))[:, None] * nlev + np.arange(nlev)[None]
      off_t = (lead_t * slab).ravel().astype(np.int64)
      off_c = off_t.copy()
      got = np.empty((nlead * nlev, 1, _lib.DET_NSTAT), np.float64)
      before = ctx.transfer_stats()['h2d_bytes']
      ctx.det_metrics(f.ctypes.data, truth.ctypes.data, clim.ctypes.data,
                      _lib.F32, off_f, off_t, off_c, spec, False,
                      got.ctypes.data, host=True)
      h2d.append(ctx.transfer_stats()['h2d_bytes'] - before)
      want = _det_device(ctx, f, truth, clim, off_f, off_t, off_c, spec, False)
      np.testing.assert_array_equal(got, want)
    st = ctx.transfer_stats()
  finally:
    ctx.set_slab_cache(0)
  full = 3 * nlead * nlev * slab * 4
  if cache_slabs == 0:
    assert all(b == full for b in h2d) and st['cache_hits'] == 0
  elif cache_slabs == 1000:
    # first chunk ships everything, later ones the forecast + one new valid time
    assert h2d[0] == full
    assert all(b == (nlead + 2) * nlev * slab * 4 for b in h2d[1:])
    assert st['cache_hits'] == 2 * (ninit - 1) * (nlead - 1) * nlev
  else:
    assert st['cache_misses'] > 0  # thrashing, but still correct


def _ens_device(ctx, x, t, m, member_stride, off_x, off_t, spec, skipna):
  """Reference result: the same operands uploaded whole, device entry."""
  from weatherbench2_b200 import _lib
  dx, dt_ = ctx.to_device(x), ctx.to_device(t)
  base = min(dx, dt_)
  n = off_x.size
  out = ctx.malloc(n * _lib.ENS_NSTAT * 8)
  try:
    ctx.ens_metrics(base, base, _lib.F32, m, member_stride,
                    off_x + (dx - base) // 4, off_t + (dt_ - base) // 4, spec,
                    skipna, out)
    return ctx.from_device(out, (n, 1, _lib.ENS_NSTAT), np.float64)
  finally:
    for p in (dx, dt_, out):
      ctx.free(p)


@pytest.mark.parametrize('cache_slabs', [0, 7, 1000])
def test_ens_host_chunk_sweep_with_slab_cache(small_stage_ctx, cache_slabs):
  """The ensemble twin of the sweep above: truth slabs repeat from chunk to
  chunk.  20 members fill 1 MiB staging with 5 fields, so a chunk of 12 fields
  runs in three groups.  With cache_slabs = 7, groups evict truth slots that
  the previous group read, so their cache fills wait for its kernel."""
  from weatherbench2_b200 import _lib
  ctx = small_stage_ctx
  m, nlat, nlon, nlead, nlev, ninit = 20, 33, 64, 4, 3, 5
  slab = nlat * nlon
  nf = nlead * nlev
  _, _, spec = _weights(ctx, nlat, nlon)
  rs = np.random.RandomState(4)
  ntime = ninit + nlead
  truth = rs.standard_normal((ntime, nlev, nlat, nlon)).astype(np.float32)
  slab_bytes = (slab + 63) // 64 * 64 * 4
  ctx.set_slab_cache(cache_slabs * slab_bytes)
  ctx.reset_transfer_stats()
  h2d = []
  try:
    for i in range(ninit):
      x = rs.standard_normal((m, nlead, nlev, nlat, nlon)).astype(np.float32)
      if i == 2:
        x[7, 1, 0, 3, 5] = np.nan
      off_x = np.arange(nf, dtype=np.int64) * slab
      lead_t = (i + np.arange(nlead))[:, None] * nlev + np.arange(nlev)[None]
      off_t = (lead_t * slab).ravel().astype(np.int64)
      got = np.empty((nf, 1, _lib.ENS_NSTAT), np.float64)
      before = ctx.transfer_stats()['h2d_bytes']
      ctx.ens_metrics_host(x.ctypes.data, truth.ctypes.data, m, nf * slab,
                           off_x, off_t, spec, False, got.ctypes.data)
      h2d.append(ctx.transfer_stats()['h2d_bytes'] - before)
      want = _ens_device(ctx, x, truth, m, nf * slab, off_x, off_t, spec,
                         False)
      np.testing.assert_array_equal(got, want)
    st = ctx.transfer_stats()
  finally:
    ctx.set_slab_cache(0)
  full = (m + 1) * nf * slab * 4
  if cache_slabs == 0:
    assert all(b == full for b in h2d) and st['cache_hits'] == 0
  elif cache_slabs == 1000:
    # first chunk ships everything, later ones the members + one new valid time
    assert h2d[0] == full
    assert all(b == (m * nlead + 1) * nlev * slab * 4 for b in h2d[1:])
    assert st['cache_hits'] == (ninit - 1) * (nlead - 1) * nlev
    assert st['cache_misses'] == (nlead + ninit - 1) * nlev
  else:
    assert st['cache_misses'] > 0  # thrashing, but still correct


def test_ens_host_matches_device_entry_and_oracle(small_stage_ctx):
  from weatherbench2_b200 import _lib
  ctx = small_stage_ctx
  m, nf, nlat, nlon = 10, 7, 33, 64
  slab = nlat * nlon
  lat, lon, spec = _weights(ctx, nlat, nlon)
  rs = np.random.RandomState(1)
  x = rs.standard_normal((m, nf, nlat, nlon)).astype(np.float32)
  t = rs.standard_normal((nf, nlat, nlon)).astype(np.float32)
  x[3, 2, 4, 4] = np.nan
  off = np.arange(nf, dtype=np.int64) * slab
  for skipna in (False, True):
    for cache in (0, 64 << 20):
      ctx.set_slab_cache(cache)
      try:
        got = np.empty((nf, 1, _lib.ENS_NSTAT), np.float64)
        for _ in range(2):  # second pass: truth slabs come from the cache
          ctx.ens_metrics_host(x.ctypes.data, t.ctypes.data, m, nf * slab, off,
                               off, spec, skipna, got.ctypes.data)
      finally:
        ctx.set_slab_cache(0)
      dx, dt_ = ctx.to_device(x), ctx.to_device(t)
      base = min(dx, dt_)
      out = ctx.malloc(nf * _lib.ENS_NSTAT * 8)
      try:
        ctx.ens_metrics(base, base, _lib.F32, m, nf * slab,
                        off + (dx - base) // 4, off + (dt_ - base) // 4, spec,
                        skipna, out)
        want = ctx.from_device(out, (nf, 1, _lib.ENS_NSTAT), np.float64)
      finally:
        for p in (dx, dt_, out):
          ctx.free(p)
      np.testing.assert_array_equal(got, want)
  fd = ('realization', 'b', 'latitude', 'longitude')
  crps, _ = orc.crps(x, fd, t, fd[1:], 'realization', lat, lon, skipna=True)
  g = got[:, 0]
  np.testing.assert_allclose(g[:, 0] / g[:, 5] - 0.5 * g[:, 1] / g[:, 6], crps,
                             rtol=1e-5)


def test_regrid_conservative_host_is_bit_identical_to_device_entry(small_stage_ctx):
  from weatherbench2_b200 import regridding as rg
  ctx = small_stage_ctx
  src = rg.Grid.from_degrees(np.linspace(0, 360, 72, endpoint=False),
                             np.linspace(-90, 90, 37))
  tgt = rg.Grid.from_degrees(np.linspace(0, 360, 24, endpoint=False),
                             np.linspace(-90, 90, 13))
  r = rg.ConservativeRegridder(src, tgt)
  rs = np.random.RandomState(2)
  nf = 301  # 1 MiB staging holds ~ 80 fields: several groups, ragged tail
  x = rs.standard_normal((nf, 72, 37)).astype(np.float32)
  x[5, 10:14, 3:9] = np.nan
  got = np.empty((nf, 24, 13), np.float32)
  lon_w, lat_w = r._weights  # pylint: disable=protected-access
  ctx.regrid_conservative_host(x.ctypes.data, got.ctypes.data, nf, 72 * 37,
                               24 * 13, lon_w, lat_w)
  dsrc = ctx.to_device(x)
  ddst = ctx.malloc(nf * 24 * 13 * 4)
  try:
    r.regrid_device(ctx, dsrc, ddst, nf)
    want = ctx.from_device(ddst, (nf, 24, 13), np.float32)
  finally:
    ctx.free(dsrc)
    ctx.free(ddst)
  np.testing.assert_array_equal(got, want)
  ref = orc.conservative_regrid(x[:9], orc.Grid(np.asarray(src.longitudes),
                                                np.asarray(src.latitudes)),
                                orc.Grid(np.asarray(tgt.longitudes),
                                         np.asarray(tgt.latitudes)))
  np.testing.assert_allclose(got[:9], ref, rtol=1e-5, atol=1e-6)
  st = ctx.transfer_stats()
  assert st['h2d_bytes'] >= x.nbytes and st['d2h_bytes'] >= got.nbytes


@pytest.mark.parametrize('ncol', [240, 72])
def test_spectrum_host_entries_match_device_entries(small_stage_ctx, ncol):
  """Per-time spectra, the time sum (accumulator stays in HBM) and the
  latitude-reduced form; 240 longitudes take the PFA kernel, 72 the Stockham
  kernel + row sum."""
  ctx = small_stage_ctx
  nrow, ntime, nslot = 19, 6, 5
  nk = ncol // 2 + 1
  rs = np.random.RandomState(3)
  x = rs.standard_normal((ntime * nslot, nrow, ncol)).astype(np.float32)
  scale = np.cos(np.deg2rad(np.linspace(-80, 80, nrow))) * 4.0e7
  dx = ctx.to_device(x)
  dout = ctx.malloc(x.shape[0] * nrow * nk * 4)
  try:
    # per time
    ctx.zonal_spectrum(dx, x.shape[0], nrow, ncol, scale, dout)
    want = ctx.from_device(dout, (x.shape[0], nrow, nk), np.float32)
    got = np.empty_like(want)
    ctx.zonal_spectrum_host(x.ctypes.data, x.shape[0], nrow, ncol, scale,
                            got.ctypes.data)
    np.testing.assert_array_equal(got, want)
    # time sum
    ctx.lib.wb2_memset(ctx.handle, dout, 0, nslot * nrow * nk * 4)
    ctx.zonal_spectrum(dx, x.shape[0], nrow, ncol, scale, dout, True, nslot)
    want = ctx.from_device(dout, (nslot, nrow, nk), np.float32)
    got = np.empty_like(want)
    ctx.zonal_spectrum_host(x.ctypes.data, x.shape[0], nrow, ncol, scale,
                            got.ctypes.data, True, nslot)
    # groups of time steps are added in a different association than one
    # launch over all time steps: equal to rounding, not bit for bit
    np.testing.assert_allclose(got, want, rtol=2e-6)
    # latitude-reduced
    ctx.zonal_spectrum_latsum(dx, x.shape[0], nrow, ncol, scale, dout, nslot)
    want = ctx.from_device(dout, (nslot, nk), np.float32)
    got = np.empty_like(want)
    ctx.zonal_spectrum_latsum_host(x.ctypes.data, x.shape[0], nrow, ncol,
                                   scale, got.ctypes.data, nslot)
    np.testing.assert_allclose(got, want, rtol=2e-6)
  finally:
    ctx.free(dx)
    ctx.free(dout)


def test_operators_with_numpy_inputs_use_the_streaming_entries():
  """CRPS / regrid / spectrum operators on NumPy data == on CUDA tensors."""
  import torch
  from weatherbench2_b200 import (_lib, derived_variables as dvs, metrics,
                                  regridding as rg, xarray_lite as xl)
  ctx = _lib.default_context()
  rs = np.random.RandomState(4)
  nlat, nlon = 37, 72
  lat = np.linspace(-90, 90, nlat)
  lon = np.linspace(0, 360, nlon, endpoint=False)
  dims = ('time', 'latitude', 'longitude')
  x = rs.standard_normal((6, 3) + (nlat, nlon)).astype(np.float32)
  t = rs.standard_normal((3, nlat, nlon)).astype(np.float32)
  coords = {'time': np.arange(3), 'latitude': lat, 'longitude': lon}
  xh = xl.Dataset({'z': (('realization',) + dims, x)},
                  dict(coords, realization=np.arange(6)))
  th = xl.Dataset({'z': (dims, t)}, coords)
  xd = xl.Dataset({'z': (('realization',) + dims, torch.from_numpy(x).cuda())},
                  dict(coords, realization=np.arange(6)))
  td = xl.Dataset({'z': (dims, torch.from_numpy(t).cuda())}, coords)
  ctx.reset_transfer_stats()
  a = metrics.CRPS().compute_chunk(xh, th)['z'].values
  assert ctx.transfer_stats()['h2d_bytes'] == x.nbytes + t.nbytes
  b = metrics.CRPS().compute_chunk(xd, td)['z'].values
  np.testing.assert_array_equal(a, b)
  want, _ = orc.crps(x, ('realization',) + dims, t, dims, 'realization', lat,
                     lon)
  np.testing.assert_allclose(a, want, rtol=1e-5, atol=1e-6)
  # spectrum
  sh = dvs.ZonalEnergySpectrum('z').compute(th)
  sd = dvs.ZonalEnergySpectrum('z').compute(td)
  np.testing.assert_array_equal(sh.values, _np(sd.values))
  sh = dvs.ZonalEnergySpectrum('z').compute(th, time_sum_dim='time')
  sd = dvs.ZonalEnergySpectrum('z').compute(td, time_sum_dim='time')
  np.testing.assert_allclose(sh.values, _np(sd.values), rtol=2e-6)
  # regrid (lon, lat layout)
  src = rg.Grid.from_degrees(lon, lat)
  tgt = rg.Grid.from_degrees(np.linspace(0, 360, 24, endpoint=False),
                             np.linspace(-90, 90, 13))
  y = rs.standard_normal((5, nlon, nlat)).astype(np.float32)
  r = rg.ConservativeRegridder(src, tgt)
  np.testing.assert_array_equal(
      r.regrid_array(y), _np(r.regrid_array(torch.from_numpy(y).cuda())))


def test_gathered_host_operand_uploads_only_referenced_slabs():
  """SpatialMSE against a by-init truth gather of a long record: the map
  kernels have no streaming entry, so the operand is uploaded -- but only the
  slabs the gather references (ADVICE r1: the whole record was uploaded)."""
  from weatherbench2_b200 import (_lib, _spatial as sp, evaluation, metrics,
                                  xarray_lite as xl)
  rs = np.random.RandomState(5)
  nlat, nlon, ninit, nlead, ntime = 19, 36, 2, 3, 400
  lat = np.linspace(-90, 90, nlat)
  lon = np.linspace(0, 360, nlon, endpoint=False)
  times = (np.datetime64('2020-01-01', 'ns') +
           np.arange(ntime) * np.timedelta64(1, 'D'))
  lead = np.arange(nlead) * np.timedelta64(1, 'D').astype('timedelta64[ns]')
  init = times[200:200 + ninit]
  f = rs.standard_normal((ninit, nlead, nlat, nlon)).astype(np.float32)
  t = rs.standard_normal((ntime, nlat, nlon)).astype(np.float32)
  forecast = xl.Dataset(
      {'z': (('init_time', 'lead_time', 'latitude', 'longitude'), f)},
      {'init_time': init, 'lead_time': lead, 'latitude': lat, 'longitude': lon,
       'valid_time': (('init_time', 'lead_time'),
                      init[:, None] + lead[None, :])})
  truth = xl.Dataset({'z': (('time', 'latitude', 'longitude'), t)},
                     {'time': times, 'latitude': lat, 'longitude': lon})
  tr = evaluation.select_truth_at_valid_time(truth, forecast)
  uploaded = []
  ctx = _lib.default_context()
  orig = ctx.to_device
  ctx.to_device = lambda a: (uploaded.append(np.asarray(a).nbytes), orig(a))[1]
  try:
    got = metrics.SpatialMSE().compute_chunk(forecast, tr)['z'].values
  finally:
    ctx.to_device = orig
  idx = 200 + np.arange(ninit)[:, None] + np.arange(nlead)[None, :]
  np.testing.assert_allclose(got, (f - t[idx]) ** 2, rtol=1e-6)
  assert sum(uploaded) < 3 * f.nbytes  # not the 400-step record (54 x larger)
  assert sp is not None

"""GPU parity tests of the prime-factor / row-pair / TMA spectrum kernel
(csrc/spectrum_pfa.cu) through the raw C ABI: per-time spectra, the device-side
time sum and the fused latitude-weighted meridional reduction
(wb2_zonal_spectrum_latsum), against NumPy's float64 rfft -- the reference's
own arithmetic (weatherbench2/derived_variables.py:592-626) -- and against the
Stockham kernels of csrc/spectrum.cu."""
import numpy as np
import pytest

from oracle import wb2_oracle as orc

pytestmark = pytest.mark.gpu

R_EARTH = 1000 * (6357 + 6378) / 2


def _want(x, scale):
  """[field][row][k] float64: |rfft(norm=forward)|^2 * (1, 2, 2, ...) * scale."""
  f = np.fft.rfft(x.astype(np.float64), axis=-1, norm='forward')
  s = (f * np.conj(f)).real
  s[..., 1:] *= 2
  return s * scale[None, :, None]


def _run(ctx, x, scale, accumulate=False, nslot=0):
  nfield, nrow, ncol = x.shape
  nk = ncol // 2 + 1
  nout = nslot if accumulate else nfield
  src = ctx.to_device(x)
  dst = ctx.malloc(nout * nrow * nk * 4)
  try:
    ctx.lib.wb2_memset(ctx.handle, dst, 0, nout * nrow * nk * 4)
    ctx.zonal_spectrum(src, nfield, nrow, ncol, scale, dst, accumulate, nslot)
    return ctx.from_device(dst, (nout, nrow, nk), np.float32).astype(np.float64)
  finally:
    ctx.free(src)
    ctx.free(dst)


def _run_latsum(ctx, x, scale, nslot):
  nfield, nrow, ncol = x.shape
  nk = ncol // 2 + 1
  src = ctx.to_device(x)
  dst = ctx.malloc(nslot * nk * 4)
  try:
    ctx.zonal_spectrum_latsum(src, nfield, nrow, ncol, scale, dst, nslot)
    return ctx.from_device(dst, (nslot, nk), np.float32).astype(np.float64)
  finally:
    ctx.free(src)
    ctx.free(dst)


def _check(got, want, tol=1e-5):
  power = want.sum(axis=-1, keepdims=True)
  np.testing.assert_allclose(got.sum(axis=-1), want.sum(axis=-1), rtol=tol)
  assert np.max(np.abs(got - want) / power) < tol


def _case(nfield, nrow, ncol, seed, offset=0.0):
  rs = np.random.RandomState(seed)
  x = (rs.standard_normal((nfield, nrow, ncol)) + offset).astype(np.float32)
  lat = np.linspace(-90, 90, nrow) if nrow > 1 else np.array([10.0])
  scale = np.cos(np.deg2rad(lat)) * 2 * np.pi * R_EARTH + 1.0  # > 0 at the poles
  return x, scale


@pytest.mark.parametrize('ncol', [1440, 720, 240])
@pytest.mark.parametrize('nrow', [1, 2, 5, 6, 7, 23, 40])
def test_pfa_per_time_spectra_match_rfft(monkeypatch, ncol, nrow):
  """Ragged row counts: odd (a padding row in the last pair), fewer rows than a
  group, exactly one group, several groups."""
  from weatherbench2_b200 import _lib
  monkeypatch.setenv('WB2_SPECTRUM_PATH', 'pfa')  # fails if PFA is not eligible
  ctx = _lib.default_context()
  x, scale = _case(5, nrow, ncol, seed=ncol + nrow, offset=1.5)
  got = _run(ctx, x, scale)
  _check(got, _want(x, scale))


@pytest.mark.parametrize('ncol', [1440, 240])
def test_pfa_equals_stockham_kernels(monkeypatch, ncol):
  from weatherbench2_b200 import _lib
  ctx = _lib.default_context()
  x, scale = _case(4, 37, ncol, seed=5)
  res = {}
  for path in ('pfa', 'fixed', 'generic'):
    monkeypatch.setenv('WB2_SPECTRUM_PATH', path)
    res[path] = _run(ctx, x, scale)
  want = _want(x, scale)
  power = want.sum(axis=-1, keepdims=True)
  for path in ('fixed', 'generic'):
    assert np.max(np.abs(res['pfa'] - res[path]) / power) < 2e-6


@pytest.mark.parametrize('ncol,nrow', [(1440, 33), (720, 11), (240, 50)])
def test_pfa_time_sum_matches_sum_of_spectra(monkeypatch, ncol, nrow):
  """accumulate=1: field i is added to slot i % nslot (the device-side time sum
  of scripts/compute_zonal_energy_spectrum.py:234); deterministic."""
  from weatherbench2_b200 import _lib
  monkeypatch.setenv('WB2_SPECTRUM_PATH', 'pfa')
  ctx = _lib.default_context()
  ntime, nslot = 7, 3
  x, scale = _case(ntime * nslot, nrow, ncol, seed=11)
  got = _run(ctx, x, scale, accumulate=True, nslot=nslot)
  want = _want(x, scale).reshape(ntime, nslot, nrow, -1).sum(axis=0)
  _check(got, want)
  again = _run(ctx, x, scale, accumulate=True, nslot=nslot)
  np.testing.assert_array_equal(got, again)


@pytest.mark.parametrize('ncol,nrow', [(1440, 721), (1440, 9), (720, 361), (240, 121),
                                       (64, 33), (360, 19)])
def test_latsum_matches_weighted_mean_of_the_reference_spectrum(ncol, nrow):
  """North star: rFFT along longitude followed by a weighted meridional
  reduction.  Parity: the get_lat_weights-weighted latitude mean
  (weatherbench2/metrics.py:40-60) of the reference's per-latitude spectrum
  (derived_variables.py:592-626), both from the oracle.  64 and 360 longitudes
  take the fallback (Stockham kernel + row sum)."""
  from weatherbench2_b200 import _lib
  ctx = _lib.default_context()
  ntime, nslot = 3, 2
  rs = np.random.RandomState(ncol)
  x = (rs.standard_normal((ntime * nslot, nrow, ncol)) + 0.5).astype(np.float32)
  lat = np.linspace(-90, 90, nrow)
  lon = np.linspace(0, 360, ncol, endpoint=False)
  spec, sd, _, _ = orc.zonal_energy_spectrum(
      x, ('time', 'latitude', 'longitude'), lat, lon)
  assert sd == ('time', 'latitude', 'zonal_wavenumber')
  w = orc.get_lat_weights(lat)  # mean(w) == 1
  want = (spec * w[None, :, None]).sum(axis=1) / w.sum()          # lat mean
  want = want.reshape(ntime, nslot, -1).mean(axis=0)              # time mean
  scale = orc.circumference(lat) * w / w.sum() / ntime
  got = _run_latsum(ctx, x, scale, nslot)
  np.testing.assert_allclose(got, want, rtol=2e-5,
                             atol=1e-6 * want.sum(axis=-1).max())
  np.testing.assert_allclose(got.sum(axis=-1), want.sum(axis=-1), rtol=1e-5)


def test_latsum_latitude_band(monkeypatch):
  """A latitude band = zero weights outside it (the lat-band spectra of the
  WB2 paper); rows with zero weight contribute nothing."""
  from weatherbench2_b200 import _lib
  monkeypatch.setenv('WB2_SPECTRUM_PATH', 'pfa')
  ctx = _lib.default_context()
  nrow, ncol = 181, 1440
  rs = np.random.RandomState(3)
  x = rs.standard_normal((2, nrow, ncol)).astype(np.float32)
  lat = np.linspace(-90, 90, nrow)
  band = (np.abs(lat) >= 30) & (np.abs(lat) <= 60)
  w = orc.get_lat_weights(lat) * band
  circ = orc.circumference(lat)
  want = (_want(x, circ) * w[None, :, None]).sum(axis=1) / w.sum()
  got = _run_latsum(ctx, x, circ * w / w.sum(), 2)
  np.testing.assert_allclose(got, want, rtol=2e-5,
                             atol=1e-6 * want.sum(axis=-1).max())


def test_pfa_full_size_parseval(monkeypatch):
  """configs[4] shape (721 x 1440): total power == mean square of the row
  (+ the doubled Nyquist term), every row, through the PFA kernel."""
  from weatherbench2_b200 import _lib
  monkeypatch.setenv('WB2_SPECTRUM_PATH', 'pfa')
  ctx = _lib.default_context()
  rs = np.random.RandomState(0)
  x = rs.standard_normal((3, 721, 1440)).astype(np.float32)
  scale = np.ones(721)
  got = _run(ctx, x, scale)
  xd = x.astype(np.float64)
  nyq = (xd[..., 0::2].sum(-1) - xd[..., 1::2].sum(-1)) / 1440
  np.testing.assert_allclose(got.sum(-1), (xd ** 2).mean(-1) + nyq ** 2, rtol=1e-5)
  _check(got[:1], _want(x[:1], scale))

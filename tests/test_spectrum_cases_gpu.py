"""Zonal-spectrum kernels (K4) bin by bin on the cases of tests/spectrum_cases.py:
every bin within the per-bin bound of DESIGN K4 at realistic magnitudes and
slopes, structural rows to their exact answers, NaN / inf confined to their
rows, zero-weight rows skipped by the latitude reduction, on every path (PFA
at 1440 / 720 / 240, fixed and generic Stockham, the unaligned fallback and
the Stockham-only sizes) and through the host-buffer entries."""
import numpy as np
import pytest

import spectrum_cases as sc
from oracle import wb2_oracle as orc

pytestmark = pytest.mark.gpu


def _ctx():
  from weatherbench2_b200 import _lib
  return _lib.default_context()


def _spectra(ctx, x, scale, accumulate=False, nslot=0, unaligned=False):
  """wb2_zonal_spectrum on device buffers; `unaligned` offsets the base by 8 B
  (not 16-byte aligned: the PFA kernel's TMA rows decline it)."""
  nfield, nrow, ncol = x.shape
  nk = ncol // 2 + 1
  nout = nslot if accumulate else nfield
  off = 8 if unaligned else 0
  src = ctx.malloc(x.nbytes + 16)
  dst = ctx.malloc(nout * nrow * nk * 4)
  try:
    from weatherbench2_b200._lib import _P, check
    x = np.ascontiguousarray(x)
    check(ctx.lib.wb2_memcpy_h2d(ctx.handle, _P(src + off), _P(x.ctypes.data), x.nbytes))
    ctx.lib.wb2_memset(ctx.handle, dst, 0, nout * nrow * nk * 4)
    ctx.zonal_spectrum(src + off, nfield, nrow, ncol, scale, dst, accumulate, nslot)
    return ctx.from_device(dst, (nout, nrow, nk), np.float32)
  finally:
    ctx.free(src)
    ctx.free(dst)


def _latsum(ctx, x, scale, nslot):
  nfield, nrow, ncol = x.shape
  nk = ncol // 2 + 1
  src = ctx.to_device(x)
  dst = ctx.malloc(nslot * nk * 4)
  try:
    ctx.zonal_spectrum_latsum(src, nfield, nrow, ncol, scale, dst, nslot)
    return ctx.from_device(dst, (nslot, nk), np.float32)
  finally:
    ctx.free(src)
    ctx.free(dst)


def _spectra_host(ctx, x, scale, accumulate=False, nslot=0):
  nfield, nrow, ncol = x.shape
  nout = nslot if accumulate else nfield
  out = np.zeros((nout, nrow, ncol // 2 + 1), np.float32)
  ctx.zonal_spectrum_host(x.ctypes.data, nfield, nrow, ncol, scale, out.ctypes.data,
                          accumulate, nslot)
  return out


def _latsum_host(ctx, x, scale, nslot):
  out = np.zeros((nslot, x.shape[-1] // 2 + 1), np.float32)
  ctx.zonal_spectrum_latsum_host(x.ctypes.data, x.shape[0], x.shape[1], x.shape[2], scale,
                                 out.ctypes.data, nslot)
  return out


def _check(got, x, scale, path, nacc=1, summed_over=None):
  """Every bin of got [field][row][k] within the bound; `summed_over`: the
  leading axis of x that got is a sum over (with its bound summed)."""
  b, w = sc.bound(x, scale, path)
  if summed_over is not None:
    b = b.sum(axis=summed_over) + (nacc - 1) * sc.U * np.abs(w).sum(axis=summed_over)
    w = w.sum(axis=summed_over)
  got = got.astype(np.float64)
  assert np.isfinite(got).all()
  err = np.abs(got - w)
  ratio = np.divide(err, b, out=np.where(err == 0, 0.0, np.inf), where=b > 0)
  worst = np.unravel_index(np.argmax(ratio), ratio.shape)
  assert ratio.max() <= 1.0, (f'{path}: bin {worst} got {got[worst]!r} want {w[worst]!r} '
                              f'bound {b[worst]!r} ({ratio.max():.3g} x)')


def _scale(nrow):
  lat = np.linspace(-89, 89, nrow) if nrow > 1 else np.array([30.0])
  return orc.circumference(lat)


# ---- realistic rows, every path -----------------------------------------------
@pytest.mark.parametrize('kind', sc.REALISTIC)
@pytest.mark.parametrize('ncol,path', [(1440, 'pfa'), (720, 'pfa'), (240, 'pfa'),
                                       (1440, 'fixed'), (1440, 'generic'),
                                       (720, 'generic'), (240, 'fixed')])
def test_realistic_rows_bin_by_bin(monkeypatch, kind, ncol, path):
  monkeypatch.setenv('WB2_SPECTRUM_PATH', path)
  nrow = 7
  x = np.stack([sc.realistic(kind, nrow, ncol, seed=s) for s in (1, 2)])
  scale = _scale(nrow)
  _check(_spectra(_ctx(), x, scale), x, scale, path)


@pytest.mark.parametrize('kind', ['z500', 'temperature', 'pressure', 'humidity'])
@pytest.mark.parametrize('ncol', [1440, 720, 240])
def test_unaligned_base_falls_back_to_stockham(monkeypatch, kind, ncol):
  monkeypatch.delenv('WB2_SPECTRUM_PATH', raising=False)
  x = sc.realistic(kind, 5, ncol, seed=4)[None]
  scale = _scale(5)
  got = _spectra(_ctx(), x, scale, unaligned=True)
  _check(got, x, scale, sc.path_for(ncol, aligned=False))


@pytest.mark.parametrize('ncol', [2, 4, 12, 18, 36, 64, 360, 512])
@pytest.mark.parametrize('kind', ['z500', 'temperature', 'wind', 'humidity'])
def test_stockham_only_sizes(monkeypatch, ncol, kind):
  monkeypatch.delenv('WB2_SPECTRUM_PATH', raising=False)
  x = sc.realistic(kind, 3, ncol, seed=ncol)[None]
  scale = _scale(3)
  _check(_spectra(_ctx(), x, scale), x, scale, sc.path_for(ncol))


@pytest.mark.parametrize('nrow', [1, 2, 9, 4, 721])
def test_row_counts(monkeypatch, nrow):
  """1, 2, an odd count, one G-group at 1440 (G = 2: 4 rows) and 721."""
  monkeypatch.setenv('WB2_SPECTRUM_PATH', 'pfa')
  x = sc.realistic('z500_tapered', nrow, 1440, seed=nrow)[None]
  scale = _scale(nrow)
  _check(_spectra(_ctx(), x, scale), x, scale, 'pfa')


@pytest.mark.parametrize('ncol', [1440, 240, 512])
def test_long_time_sum(monkeypatch, ncol):
  """A few rows x 1460 time steps (a year of 6-hourly fields) summed per bin:
  bounds the same-sign float32 accumulation term; the host entry gives the
  same bits."""
  monkeypatch.delenv('WB2_SPECTRUM_PATH', raising=False)
  ntime, nrow = 1460, 3
  x = np.stack([sc.realistic('temperature', nrow, ncol, seed=t) for t in range(ntime)])
  scale = _scale(nrow)
  ctx = _ctx()
  got = _spectra(ctx, x, scale, accumulate=True, nslot=1)
  _check(got, x, scale, sc.path_for(ncol), nacc=ntime, summed_over=0)
  np.testing.assert_array_equal(_spectra_host(ctx, x, scale, True, 1), got)
  # latitude reduction over the same fields: rows x time steps per bin
  w = orc.get_lat_weights(np.linspace(-60, 60, nrow))
  lsc = scale * w / w.sum() / ntime
  red = _latsum(ctx, x, lsc, 1).astype(np.float64)
  b, want = sc.bound(x, lsc, sc.path_for(ncol))
  b = b.sum(axis=(0, 1)) + ntime * nrow * sc.U * np.abs(want).sum(axis=(0, 1))
  want = want.sum(axis=(0, 1))
  assert (np.abs(red[0] - want) <= b).all()
  np.testing.assert_array_equal(_latsum_host(ctx, x, lsc, 1), red.astype(np.float32))


# ---- structural rows ----------------------------------------------------------
@pytest.mark.parametrize('ncol,path', [(1440, 'pfa'), (720, 'pfa'), (240, 'pfa'),
                                       (1440, 'fixed'), (1440, 'generic'), (12, 'generic'),
                                       (64, 'fixed'), (2, 'generic')])
def test_structural_rows_exact(monkeypatch, ncol, path):
  monkeypatch.setenv('WB2_SPECTRUM_PATH', path)
  cases = sc.structural(ncol)
  x = np.stack([row for _, row, _ in cases])[None]
  got = _spectra(_ctx(), x, np.ones(len(cases)))[0].astype(np.float64)
  for (name, _, exact), g in zip(cases, got):
    if name in ('constant', 'zeros', 'signed_zeros'):
      assert (g[1:] == 0).all(), f'{name}: non-DC bins {g[1:][g[1:] != 0][:4]}'
      np.testing.assert_allclose(g[0], exact[0], rtol=4 * sc.U, err_msg=name)
    else:
      np.testing.assert_allclose(g, exact, rtol=16 * sc.U, atol=1e-6 * exact.max(),
                                 err_msg=name)


@pytest.mark.parametrize('ncol,path', [(1440, 'pfa'), (720, 'pfa'), (240, 'pfa'),
                                       (1440, 'fixed'), (1440, 'generic')])
def test_pure_tones_land_in_their_bin(monkeypatch, ncol, path):
  """Tones at 1, N/2 - 1, Nyquist and one bin of every residue class of the
  Good-Thomas output map: every stage-C task and its mirror produce a known
  bin, and nothing leaks elsewhere beyond the bound."""
  monkeypatch.setenv('WB2_SPECTRUM_PATH', path)
  bins = sc.tone_bins(ncol)
  x = np.stack([250.0 + sc.tone(ncol, p, amp=7.0) for p in bins]).astype(np.float32)[None]
  scale = np.ones(len(bins))
  got = _spectra(_ctx(), x, scale)
  _check(got, x, scale, path)
  g = got[0].astype(np.float64)
  for i, p in enumerate(bins):
    others = np.delete(g[i], [0, p])
    assert g[i, p] > 1e6 * max(others.max(), 1e-30) or others.max() == 0, p


# ---- NaN / inf ----------------------------------------------------------------
@pytest.mark.parametrize('ncol', [1440, 720, 240])
@pytest.mark.parametrize('bad', [np.nan, np.inf, -np.inf])
@pytest.mark.parametrize('where', ['row_a', 'row_b', 'first_pair_of_group',
                                   'last_pair_of_group', 'last_odd_row'])
def test_nonfinite_stays_in_its_row(monkeypatch, ncol, bad, where):
  """A single NaN / inf makes every bin of its own row non-finite, as in the
  oracle (which bins are NaN and which inf depends on the FFT's order of
  operations), and nothing else: the other row of the pair, the neighbouring
  rows and the other field stay within the bound."""
  monkeypatch.setenv('WB2_SPECTRUM_PATH', 'pfa')
  nrow, rows = sc.nonfinite_rows(ncol)
  row = rows[where]
  x = np.stack([sc.realistic('z500', nrow, ncol, seed=s) for s in (5, 6)])
  x[0, row, 17] = bad
  scale = _scale(nrow)
  ctx = _ctx()
  got = _spectra(ctx, x, scale).astype(np.float64)
  want = sc.want(x[0, row:row + 1], scale[row:row + 1])
  assert not np.isfinite(want).any() and not np.isfinite(got[0, row]).any()
  keep = np.ones((2, nrow), bool)
  keep[0, row] = False
  b, w = sc.bound(x, scale, 'pfa')
  assert (np.abs(got[keep] - w[keep]) <= b[keep]).all()
  # the latitude reduction: the bad row has nonzero weight -> non-finite bins,
  # the other field untouched
  red = _latsum(ctx, x, scale / nrow, 2)
  assert not np.isfinite(red[0]).any() and np.isfinite(red[1]).all()


@pytest.mark.parametrize('ncol', [1440, 720, 240, 360])
@pytest.mark.parametrize('bad', [np.nan, np.inf])
@pytest.mark.parametrize('host', [False, True])
def test_latitude_band_ignores_rows_outside_it(ncol, bad, host):
  """compute_latitude_mean(lat_slice=...) zeroes the weights outside the band;
  NaN / inf rows there (including the last row of an odd nrow, which the PFA
  padding row repeats) must not reach the band mean.  Equal to the oracle's
  weighted mean over the selected rows only.  360 longitudes take the
  Stockham fallback and its row sum."""
  from weatherbench2_b200 import derived_variables as dvs
  from weatherbench2_b200 import xarray_lite as xl
  nrow = 37
  lat = np.linspace(-90, 90, nrow)
  lon = np.linspace(0, 360, ncol, endpoint=False)
  x = np.stack([sc.realistic('temperature', nrow, ncol, seed=s) for s in (7, 8)])
  x[:, 0, 3] = bad           # south pole row, outside the band
  x[:, nrow - 1, 5] = bad    # last (odd) row, outside the band
  x[1, 2, :] = bad           # a whole row outside the band
  band = slice(-40, 55)
  dims = ('time', 'latitude', 'longitude')
  ds = xl.Dataset({'t': (dims, x)}, {'time': np.arange(2), 'latitude': lat,
                                     'longitude': lon})
  if host:
    got = dvs.ZonalEnergySpectrum('t').compute_latitude_mean(ds, lat_slice=band).values
  else:
    import torch
    dsg = xl.Dataset({'t': (dims, torch.from_numpy(x).cuda())},
                     {'time': np.arange(2), 'latitude': lat, 'longitude': lon})
    got = dvs.ZonalEnergySpectrum('t').compute_latitude_mean(dsg, lat_slice=band).values
    got = got.cpu().numpy() if isinstance(got, torch.Tensor) else got
  got = np.asarray(got, np.float64)
  sel = (lat >= band.start) & (lat <= band.stop)
  w = orc.get_lat_weights(lat) * sel
  spec, _, _, _ = orc.zonal_energy_spectrum(x[:, sel].astype(np.float64), dims, lat[sel], lon)
  want = (spec * w[sel][None, :, None]).sum(axis=1) / w.sum()
  assert np.isfinite(got).all()
  lsc = orc.circumference(lat) * w / w.sum()
  b, _ = sc.bound(x[:, sel], lsc[sel], sc.path_for(ncol))
  b = b.sum(axis=1) + sel.sum() * sc.U * np.abs(want)
  assert (np.abs(got - want) <= b).all(), np.max(np.abs(got - want) / b)


def test_overflowing_row_in_padding_source_stays_inf(monkeypatch):
  """An odd nrow whose last row's power overflows float32 (+inf at bin 0):
  the latitude sum is +inf there, not 0 * inf = NaN from the padding row that
  repeats it."""
  monkeypatch.setenv('WB2_SPECTRUM_PATH', 'pfa')
  nrow, ncol = 5, 1440
  x = sc.realistic('wind', nrow, ncol, seed=9)[None]
  x[0, nrow - 1] = np.float32(1e25)
  red = _latsum(_ctx(), x, np.ones(nrow), 1)[0]
  assert red[0] == np.inf
  assert np.isfinite(red[1:]).all()


# ---- host entries -------------------------------------------------------------
@pytest.mark.parametrize('ncol', [1440, 720, 240, 360, 64])
def test_host_entries_bit_identical(monkeypatch, ncol):
  monkeypatch.delenv('WB2_SPECTRUM_PATH', raising=False)
  ntime, nslot, nrow = 3, 2, 11
  x = np.stack([sc.realistic('z500', nrow, ncol, seed=s) for s in range(ntime * nslot)])
  scale = _scale(nrow)
  ctx = _ctx()
  np.testing.assert_array_equal(_spectra_host(ctx, x, scale), _spectra(ctx, x, scale))
  np.testing.assert_array_equal(_spectra_host(ctx, x, scale, True, nslot),
                                _spectra(ctx, x, scale, True, nslot))
  lsc = scale / nrow / ntime
  np.testing.assert_array_equal(_latsum_host(ctx, x, lsc, nslot), _latsum(ctx, x, lsc, nslot))

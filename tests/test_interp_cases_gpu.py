"""K8 (wb2_regrid_bilinear, wb2_regrid_gather) and wb2_spectrum_interp on the
cases of interp_cases.py, through `_lib.Context` and through the public
operators on NumPy and CUDA input: bilinear bit-equal to the float32
jnp.interp model everywhere (NaN and inf included), nearest bit-equal to the
gather of the BallTree indices, spectrum interpolation equal to the float32
rounding of scipy's value (and so within its bound) with scipy's NaN / inf
pattern, padding between fields untouched, repeat calls bit-identical, and
out-of-range taps rejected."""
import numpy as np
import pytest

import interp_cases as ic

pytestmark = pytest.mark.gpu

CASES = {c.name: c for c in ic.bilinear_cases()}
SPECTRA = {c.name: c for c in ic.spectrum_cases()}
SENTINEL = np.int32(0x7fa5a5a5)  # a NaN payload no kernel produces


def _same(a, b):
  """Bit-equal away from NaN, NaN at the same cells."""
  a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
  nan = np.isnan(a)
  return (a.shape == b.shape and np.array_equal(nan, np.isnan(b)) and
          np.array_equal(a[~nan].view(np.int32), b[~nan].view(np.int32)))


def _cuda(x):
  import torch
  return torch.from_numpy(np.ascontiguousarray(x)).cuda()


@pytest.mark.parametrize('name', sorted(CASES))
def test_bilinear_bit_equal_to_jnp_interp_model(name):
  from weatherbench2_b200 import regridding
  case = CASES[name]
  want = ic.bilinear_model(case.fields, case.src, case.tgt)
  r = regridding.BilinearRegridder(case.src.grid(), case.tgt.grid())
  got = r.regrid_array(case.fields)
  assert got.dtype == np.float32 and _same(got, want)
  assert np.array_equal(np.asarray(r.regrid_array(case.fields)).view(np.int32),
                        np.asarray(got).view(np.int32))
  dev = r.regrid_array(_cuda(case.fields))
  assert dev.is_cuda and _same(dev.cpu().numpy(), want)


@pytest.mark.parametrize('name', sorted(set(CASES) - {'upsample_15_to_025'}))
def test_nearest_bit_equal_to_ball_tree_gather(name):
  from weatherbench2_b200 import regridding
  case = CASES[name]
  idx = ic.ball_tree_indices(case.src, case.tgt)
  nf = case.fields.shape[0]
  want = case.fields.reshape(nf, -1)[:, idx].reshape((nf,) + case.tgt.shape)
  r = regridding.NearestRegridder(case.src.grid(), case.tgt.grid())
  for x in (case.fields, _cuda(case.fields)):
    got = r.regrid_array(x)
    got = got.cpu().numpy() if hasattr(got, 'cpu') else got
    assert np.array_equal(got.view(np.int32), want.view(np.int32))  # payloads too


@pytest.mark.parametrize('name', ['era5_025_to_64x32', 'clamped_short_poles',
                                  'limited_area'])
def test_regrid_dataset_both_regridders(name):
  from weatherbench2_b200 import regridding, xarray_lite as xl
  case = CASES[name]
  x = np.swapaxes(case.fields, 1, 2)[:, ::-1]  # (time, lat decreasing, lon)
  ds = xl.Dataset({'x': (('time', 'latitude', 'longitude'), x)},
                  {'time': np.arange(x.shape[0]),
                   'latitude': np.asarray(case.src.latitudes)[::-1],
                   'longitude': case.src.longitudes})
  idx = ic.ball_tree_indices(case.src, case.tgt)
  nf = case.fields.shape[0]
  wants = {regridding.BilinearRegridder:
               ic.bilinear_model(case.fields, case.src, case.tgt),
           regridding.NearestRegridder:
               case.fields.reshape(nf, -1)[:, idx].reshape(
                   (nf,) + case.tgt.shape)}
  for cls, want in wants.items():
    out = cls(case.src.grid(), case.tgt.grid()).regrid_dataset(ds)['x']
    assert out.dims == ('time', 'latitude', 'longitude')
    np.testing.assert_array_equal(out.coords['latitude'].values,
                                  case.tgt.latitudes)
    assert _same(out.values, np.swapaxes(want, 1, 2))


# ---- raw ABI --------------------------------------------------------------------
def _padded(fields, stride):
  """(nfield, n) float32 -> flat buffer with `stride` elements per field, the
  padding filled with SENTINEL."""
  nf, n = fields.shape
  buf = np.full((nf, stride), SENTINEL, np.int32).view(np.float32)
  buf[:, :n] = fields
  return buf


@pytest.mark.parametrize('nfield', [65535, 65536, 65537])
def test_raw_entries_field_loop_strides_and_padding(nfield):
  from weatherbench2_b200 import _lib, regridding  # noqa: F401
  from weatherbench2_b200 import _regrid_interp as ri
  ctx = _lib.default_context(0)
  src = ic.GridSpec(np.array([0.0, 90.0, 180.0, 270.0]),
                    np.array([-60.0, 0.0, 60.0]))
  tgt = ic.GridSpec(np.array([45.0, 135.0, 300.0, 0.0, 359.0]),
                    np.array([-90.0, 30.0]))
  rs = np.random.RandomState(nfield)
  fields = (5e4 + 100 * rs.standard_normal((nfield, 4, 3))).astype(np.float32)
  fields[7, 1, 0] = np.inf        # clamped tap, right of a lerp
  fields[-1, 0, 2] = np.nan
  fields[65534 % nfield, 3, 1] = -np.inf
  ns, nt, s_stride, d_stride = 12, 10, 13, 11
  lon, lat = ri.BilinearRegridder(src.grid(), tgt.grid())._taps  # pylint: disable=protected-access
  want = ic.bilinear_model(fields, src, tgt).reshape(nfield, nt)
  assert _same(want, ic.kernel_formula(fields, lon, lat).reshape(nfield, nt))
  idx = np.array([11, 0, 0, 5, 11, 3, 3, 7, 1, 0], np.int32)
  gathered = fields.reshape(nfield, ns)[:, idx]
  d_src = _cuda(_padded(fields.reshape(nfield, ns), s_stride))
  for entry, expect in (('bilinear', want), ('gather', gathered)):
    d_dst = _cuda(np.full((nfield, d_stride), SENTINEL, np.int32).view(
        np.float32))
    for _ in range(2):  # a repeat call writes the same bits
      if entry == 'bilinear':
        ctx.regrid_bilinear(d_src.data_ptr(), d_dst.data_ptr(), nfield,
                            s_stride, d_stride, (4, 3), lon, lat)
      else:
        ctx.regrid_gather(d_src.data_ptr(), d_dst.data_ptr(), nfield, s_stride,
                          d_stride, ns, idx)
      ctx.synchronize()
      out = d_dst.cpu().numpy()
      assert (out[:, nt:].view(np.int32) == SENTINEL).all(), entry
      assert _same(out[:, :nt], expect), entry
      assert not (out[:, :nt].view(np.int32) == SENTINEL).any(), entry


def test_raw_gather_ntarget_not_a_multiple_of_256():
  from weatherbench2_b200 import _lib
  ctx = _lib.default_context(0)
  rs = np.random.RandomState(3)
  ns, nt, nf = 1000, 1000 - 233, 3
  idx = rs.randint(0, ns, nt).astype(np.int32)
  idx[:4] = [0, ns - 1, ns - 1, 0]
  x = rs.standard_normal((nf, ns)).astype(np.float32)
  d_src = _cuda(x)
  d_dst = _cuda(np.full((nf, nt + 5), SENTINEL, np.int32).view(np.float32))
  ctx.regrid_gather(d_src.data_ptr(), d_dst.data_ptr(), nf, ns, nt + 5, ns, idx)
  ctx.synchronize()
  out = d_dst.cpu().numpy()
  assert np.array_equal(out[:, :nt].view(np.int32), x[:, idx].view(np.int32))
  assert (out[:, nt:].view(np.int32) == SENTINEL).all()


@pytest.mark.parametrize('axis,bad', [('lon', -2), ('lon', 4), ('lat', -2),
                                      ('lat', 3), ('lon', -1), ('lat', -1)])
def test_raw_bilinear_rejects_taps_out_of_range(axis, bad):
  """-2 and n are out of range; -1 in only one of i0 / i1 is rejected too (a
  NaN target has both at -1)."""
  from weatherbench2_b200 import _lib
  ctx = _lib.default_context(0)
  buf = ctx.malloc(1024)
  ok = (np.array([0, 1]), np.array([1, 1]), np.float32([0.5, -1.0]))
  for which in (0, 1):
    taps = [np.array(a, copy=True) for a in ok]
    taps[which][0] = bad
    args = (taps, ok) if axis == 'lon' else (ok, taps)
    with pytest.raises(_lib.Wb2Error, match='tap 0 out of range'):
      ctx.regrid_bilinear(buf, buf, 1, 12, 4, (4, 3), *args)
  ctx.free(buf)


@pytest.mark.parametrize('bad', [-1, 12])
def test_raw_gather_rejects_indices_out_of_range(bad):
  from weatherbench2_b200 import _lib
  ctx = _lib.default_context(0)
  buf = ctx.malloc(1024)
  with pytest.raises(_lib.Wb2Error, match='out of range'):
    ctx.regrid_gather(buf, buf, 1, 12, 3, 12, np.array([0, bad, 2]))
  ctx.free(buf)


# ---- spectrum interpolation ------------------------------------------------------------
def _check_spectrum(got, case):
  with np.errstate(invalid='ignore'):
    ref = ic.scipy_reference(case)
  assert _same(got, ref.astype(np.float32))  # scipy's NaN / inf pattern exactly
  exact = ic.exact_spectrum(case)
  fin = np.isfinite(exact)
  err = np.abs(np.asarray(got, np.float64)[fin] - exact[fin].astype(np.float64))
  assert np.all(err <= ic.spectrum_bound(case)[fin])


@pytest.mark.parametrize('name', sorted(SPECTRA))
def test_spectrum_interp_raw_entry(name):
  from weatherbench2_b200 import _lib
  ctx = _lib.default_context(0)
  case = SPECTRA[name]
  nrow, nk = case.table.shape
  d_spec = _cuda(case.spec)
  import torch
  shape = (case.nfield, nrow, case.freqs.size)
  outs = []
  for _ in range(2):
    out = torch.empty(shape, dtype=torch.float32, device='cuda')
    ctx.spectrum_interp(d_spec.data_ptr(), case.nfield, nrow, nk, case.table,
                        case.freqs, out.data_ptr())
    ctx.synchronize()
    outs.append(out.cpu().numpy())
  _check_spectrum(outs[0], case)
  assert np.array_equal(outs[0].view(np.int32), outs[1].view(np.int32))
  if name == 'zonal_1440x721':  # more items than one grid-stride sweep
    assert np.prod(shape) > 132 * 16 * 256


@pytest.mark.parametrize('name', ['zonal_240x121', 'zonal_64x33', 'nk2'])
def test_interpolate_spectral_frequencies_operator(name):
  from weatherbench2_b200 import derived_variables as dvs, xarray_lite as xl
  case = SPECTRA[name]
  nrow, nk = case.table.shape
  coords = {'time': np.arange(case.nfield), 'latitude': np.arange(nrow),
            'zonal_wavenumber': np.arange(nk),
            'frequency': xl.Coord(('zonal_wavenumber', 'latitude'),
                                  case.table.T)}
  for data in (case.spec, _cuda(case.spec)):
    da = xl.DataArray(data, ('time', 'latitude', 'zonal_wavenumber'), coords,
                      'u')
    got = dvs.interpolate_spectral_frequencies(da, 'zonal_wavenumber',
                                               case.freqs)
    vals = got.values
    vals = vals.cpu().numpy() if hasattr(vals, 'cpu') else vals
    assert got.dims == ('time', 'latitude', 'frequency')
    _check_spectrum(vals, case)

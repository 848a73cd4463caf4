"""K5 TMA-staged kernel (csrc/regrid_tma.cu) against the LDG kernel
(csrc/regrid.cu, WB2_REGRID_PATH=ldg) -- bit for bit, same taps in the same
order -- and against the oracle (weatherbench2/regridding.py:502-536)."""
import numpy as np
import pytest

from oracle import wb2_oracle as orc

pytestmark = pytest.mark.gpu


def _regrid(ctx, r, x, nfield, ns, nt, src_stride=None, dst_stride=None,
            byte_shift=0):
  src_stride = src_stride or ns
  dst_stride = dst_stride or nt
  buf = np.zeros(nfield * src_stride + 8, np.float32)
  view = buf[byte_shift // 4:byte_shift // 4 + nfield * src_stride].reshape(
      nfield, src_stride)
  view[:, :ns] = x.reshape(nfield, ns)
  dsrc = ctx.to_device(buf)
  ddst = ctx.malloc(nfield * dst_stride * 4)
  try:
    ctx.lib.wb2_memset(ctx.handle, ddst, 0, nfield * dst_stride * 4)
    r.regrid_device(ctx, dsrc + byte_shift, ddst, nfield, src_stride,
                    dst_stride)
    out = ctx.from_device(ddst, (nfield, dst_stride), np.float32)
    return out[:, :nt]
  finally:
    ctx.free(dsrc)
    ctx.free(ddst)


CASES = [
    # (source lon, source lat, target lon, target lat)
    (1440, 721, 240, 121),   # headline 0.25 -> 1.5 degree
    (360, 181, 64, 32),      # non-integer ratio, pole-less target
    (72, 37, 24, 13),
    (128, 65, 30, 11),       # odd sizes: rows never 16-byte aligned
    (90, 46, 7, 5),          # very coarse target: long runs of source rows
]


@pytest.mark.parametrize('nls,nlas,nlt,nlat', CASES)
def test_tma_path_equals_ldg_path_and_oracle(monkeypatch, nls, nlas, nlt, nlat):
  from weatherbench2_b200 import _lib, regridding as rg
  ctx = _lib.default_context()
  slon = np.linspace(0, 360, nls, endpoint=False)
  slat = np.linspace(-90, 90, nlas)
  tlon = np.linspace(0, 360, nlt, endpoint=False)
  tlat = (np.linspace(-90, 90, nlat) if nlat % 2 else
          np.linspace(-87, 87, nlat))
  r = rg.ConservativeRegridder(rg.Grid.from_degrees(slon, slat),
                               rg.Grid.from_degrees(tlon, tlat))
  rs = np.random.RandomState(nls)
  nfield = 5
  x = rs.standard_normal((nfield, nls, nlas)).astype(np.float32)
  x[1, nls // 3:nls // 3 + 9, nlas // 4:nlas // 4 + 7] = np.nan  # a NaN patch
  x[2, :3, :] = np.nan                                          # at the seam
  x[3] = np.nan
  ns, nt = nls * nlas, nlt * nlat
  res = {}
  for path in ('tma', 'ldg'):
    monkeypatch.setenv('WB2_REGRID_PATH', path)
    res[path] = _regrid(ctx, r, x, nfield, ns, nt)
  np.testing.assert_array_equal(res['tma'], res['ldg'])
  want = orc.conservative_regrid(
      x, orc.Grid(slon, slat, includes_poles=True),
      orc.Grid(tlon, tlat, includes_poles=True))
  got = res['tma'].reshape(nfield, nlt, nlat)
  np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
  np.testing.assert_allclose(got, want, rtol=1e-5, atol=2e-6)


def test_padded_field_strides_and_unaligned_base(monkeypatch):
  """Field strides larger than a slab (multiple of 4: TMA path; not a multiple
  / base not 16-byte aligned: the LDG kernel takes over) give the same numbers."""
  from weatherbench2_b200 import _lib, regridding as rg
  ctx = _lib.default_context()
  slon = np.linspace(0, 360, 72, endpoint=False)
  slat = np.linspace(-90, 90, 37)
  r = rg.ConservativeRegridder(
      rg.Grid.from_degrees(slon, slat),
      rg.Grid.from_degrees(np.linspace(0, 360, 24, endpoint=False),
                           np.linspace(-90, 90, 13)))
  rs = np.random.RandomState(0)
  x = rs.standard_normal((6, 72, 37)).astype(np.float32)
  ns, nt = 72 * 37, 24 * 13
  base = _regrid(ctx, r, x, 6, ns, nt)
  for src_stride, dst_stride, shift in [(ns + 4, nt + 3, 0), (ns + 5, nt, 0),
                                        (ns, nt, 4), (ns + 8, nt + 8, 8)]:
    got = _regrid(ctx, r, x, 6, ns, nt, src_stride, dst_stride, shift)
    np.testing.assert_array_equal(got, base)

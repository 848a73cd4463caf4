"""K5 (csrc/regrid_tma.cu, csrc/regrid.cu) on the seeded cases of
regrid_cases.py through the C ABI: wb2_regrid_conservative under the default
dispatch and under WB2_REGRID_PATH=ldg, and wb2_regrid_conservative_host on a
fresh context with 1 MB of staging (one 1440x721 field per group).  Every cell
within the per-cell bound of DESIGN.md K5, the structural and inf cases exact
(NaN / inf pattern and sign, +0 outside spike footprints), TMA and LDG bit
for bit, the host entry bit for bit, repeated calls bit for bit; the kernel
each case launches is the one the path model predicts."""
import re

import numpy as np
import pytest

import regrid_cases as rc

pytestmark = pytest.mark.gpu

SENTINEL = np.array([0x7FA5A5A5], np.uint32).view(np.float32)[0]  # NaN payload


@pytest.fixture(scope='module')
def ctx():
  from weatherbench2_b200 import _lib
  return _lib.default_context()


def run_device(ctx, c, x=None, base_offset=0, src_stride=None,
               dst_stride=None):
  """(nfield, nlon_t, nlat_t) result; checks the destination padding kept
  its sentinel."""
  x = c.x if x is None else x
  nfield = x.shape[0]
  ns, nt = c.lon.n_src * c.lat.n_src, c.lon.n_tgt * c.lat.n_tgt
  src_stride = src_stride or ns
  dst_stride = dst_stride or nt
  buf = np.full(nfield * src_stride + 8, SENTINEL, np.float32)
  sh = base_offset // 4
  buf[sh:sh + nfield * src_stride].reshape(nfield, src_stride)[:, :ns] = (
      x.reshape(nfield, ns))
  dsrc = ctx.to_device(buf)
  ddst = ctx.to_device(np.full(nfield * dst_stride, SENTINEL, np.float32))
  try:
    ctx.regrid_conservative(dsrc + base_offset, ddst, nfield, src_stride,
                            dst_stride, c.lon, c.lat)
    out = ctx.from_device(ddst, (nfield, dst_stride), np.float32)
  finally:
    ctx.free(dsrc)
    ctx.free(ddst)
  pad = out[:, nt:].view(np.uint32)
  assert (pad == SENTINEL.view(np.uint32)).all(), 'destination padding written'
  return out[:, :nt].reshape(nfield, c.lon.n_tgt, c.lat.n_tgt)


def run_host(c, monkeypatch):
  """wb2_regrid_conservative_host on a fresh context with 1 MB staging."""
  from weatherbench2_b200 import _lib
  monkeypatch.setenv('WB2_STAGE_MB', '1')
  fresh = _lib.Context(0)
  try:
    x = np.ascontiguousarray(c.x)
    out = np.zeros((c.nfield, c.lon.n_tgt, c.lat.n_tgt), np.float32)
    fresh.regrid_conservative_host(x.ctypes.data, out.ctypes.data, c.nfield,
                                   x[0].size, out[0].size, c.lon, c.lat)
    fresh.synchronize()
  finally:
    fresh.close()
  return out


def same_bits(a, b):
  return np.array_equal(np.asarray(a).view(np.uint32),
                        np.asarray(b).view(np.uint32))


@pytest.mark.parametrize('name', rc.case_names())
def test_case(ctx, monkeypatch, name):
  c = rc.get_case(name)
  monkeypatch.delenv('WB2_REGRID_PATH', raising=False)
  got = run_device(ctx, c)
  bad = rc.violations(got, c.ref, zero_exact=c.zero_exact,
                      value_exact=c.value_exact)
  assert not bad, bad
  assert same_bits(run_device(ctx, c), got), 'not repeatable'
  monkeypatch.setenv('WB2_REGRID_PATH', 'ldg')
  ldg = run_device(ctx, c)
  monkeypatch.delenv('WB2_REGRID_PATH')
  assert same_bits(ldg, got), (
      f'LDG differs from the default path in {int((ldg != got).sum())} cells')
  assert same_bits(run_host(c, monkeypatch), got), 'host entry differs'


def _launched(ctx, c):
  """Template arguments of the regrid kernel one default call launches."""
  import torch
  from torch.profiler import ProfilerActivity, profile
  torch.cuda.init()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    run_device(ctx, c, x=c.x[:1])
    ctx.synchronize()
  names = {e.name for e in prof.events() if 'regrid' in e.name}
  out = set()
  for n in names:
    m = re.search(r'regrid_tma_kernel<(\d+), (\d+), (\d+)>', n)
    if m:
      out.add(f'TMA G{m[2]} DPT{m[1]} NTAP{m[3]}')
    m = re.search(r'regrid_kernel<(\d+)>', n)
    if m:
      out.add(f'LDG DPT{m[1]}')
  return out


def test_cases_launch_the_claimed_instance(ctx, monkeypatch):
  monkeypatch.delenv('WB2_REGRID_PATH', raising=False)
  wrong = []
  seen = set()
  for c in rc.all_cases():
    key = (c.claim, id(c.lon), id(c.lat))
    if c.family == 'structural' or key in seen:
      continue
    seen.add(key)
    got = _launched(ctx, c)
    if got != {c.claim}:
      wrong.append((c.name, c.claim, sorted(got)))
  assert not wrong, wrong


def test_malformed_csr_is_rejected(ctx):
  from weatherbench2_b200 import _lib
  for name, lon, lat in rc.bad_csr_pairs():
    c = rc.Case(name, lon, lat, np.zeros((1, lon.n_src, lat.n_src),
                                         np.float32), '', 'raw')
    with pytest.raises(_lib.Wb2Error, match='strictly increasing'):
      run_device(ctx, c)


def test_1025_source_latitudes_are_unsupported(ctx):
  from weatherbench2_b200 import _lib
  lon, _ = rc.raw_pair('raw-nlat1024')
  lat = rc.raw_csr(1025, [(np.array([0, 1]), np.ones(2))])
  c = rc.Case('1025', lon, lat, np.zeros((1, lon.n_src, 1025), np.float32),
              'unsupported', 'raw')
  with pytest.raises(_lib.Wb2Error, match='error -4'):
    run_device(ctx, c)


GEOMETRY = ['1440x721-240x121', '360x721-50x91', '240x121-64x32',
            '1440x721-64x32']


@pytest.mark.parametrize('name', GEOMETRY)
def test_strides_offsets_and_batches(ctx, monkeypatch, name):
  """Padded field strides (TMA when a multiple of 4 floats, LDG otherwise)
  with NaN-payload sentinels in the padding, base offsets of 4 / 8 / 12 bytes
  (LDG), and every field of a batch equal to the field regridded alone."""
  monkeypatch.delenv('WB2_REGRID_PATH', raising=False)
  c = rc.get_case(name)
  base = run_device(ctx, c)
  ns, nt = c.x[0].size, base[0].size
  for ss, ds in ((ns + 36, nt + 7), (ns + 5, nt + 1), (ns + 4, nt)):
    assert same_bits(run_device(ctx, c, src_stride=ss, dst_stride=ds), base)
  for off in (4, 8, 12):
    assert same_bits(run_device(ctx, c, base_offset=off), base), off
  for f in range(c.nfield):
    assert same_bits(run_device(ctx, c, x=c.x[f:f + 1]), base[f:f + 1]), f


def test_one_field_and_many_fields_at_headline_size(ctx, monkeypatch):
  """1 field (120 work items, fewer than the persistent CTAs) and 37 fields
  (4440 items, many rounds of the double-buffered descriptor slots): each
  field bit-equal to the same field regridded alone, and within the bound."""
  monkeypatch.delenv('WB2_REGRID_PATH', raising=False)
  c = rc.get_case('1440x721-240x121')
  rs = np.random.RandomState(37)
  x = np.concatenate([c.x] * 5)[:37].copy()
  x += rs.standard_normal((37, 1, 1)).astype(np.float32) * np.abs(x[:, :1, :1])
  many = run_device(ctx, c, x=x)
  ref = rc.reference(c.lon, c.lat, x)
  bad = rc.violations(many, ref)
  assert not bad, bad
  for f in range(37):
    assert same_bits(run_device(ctx, c, x=x[f:f + 1]), many[f:f + 1]), f

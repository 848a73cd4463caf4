"""Reindexing in time through the CUDA slab gather (csrc/slab_gather.cu):
the C ABI against NumPy bit for bit at 721x1440 with 13 and 37 levels in all
four dtype pairs, NaN slabs, misaligned offsets and odd slabs on both
kernels, slab = 1, nslab = 0, CUDA in with CUDA out, a memmap source whose
uploaded bytes are exactly the referenced slabs, a budget small enough to
force many bands and split slabs, the host-side rejection of invalid tables,
and the three operations end to end against the oracle on device tensors and
on streamed NumPy."""
import numpy as np
import pytest

import fake_ctx_reindex
from test_reindex_cpu import (CLIM_DIMS, IVT_DIMS, TRUTH_DIMS, expand_case,
                              ivt_case, prob_case)

pytestmark = pytest.mark.gpu

GRID = 721 * 1440


def _ctx():
  from weatherbench2_b200 import _lib
  return _lib, _lib.default_context()


def _code(dtype):
  from weatherbench2_b200 import _lib
  return _lib.F64 if np.dtype(dtype) == np.float64 else _lib.F32


def device_gather(src, slab, offsets, out_dtype):
  """wb2_slab_gather on a CUDA copy of `src`; returns the output as NumPy."""
  import torch
  _, ctx = _ctx()
  x = torch.from_numpy(src).cuda()
  n = np.asarray(offsets).size
  out = torch.empty((n, slab), dtype=getattr(torch, np.dtype(out_dtype).name),
                    device='cuda')
  ctx.slab_gather(x.data_ptr(), _code(src.dtype), src.size, slab, n, offsets,
                  out.data_ptr(), _code(out_dtype))
  return out.cpu().numpy()


def host_gather(src, slab, offsets, out_dtype, budget=1 << 30):
  _, ctx = _ctx()
  n = np.asarray(offsets).size
  out = np.empty((n, slab), out_dtype)
  ctx.slab_gather_host(src.ctypes.data, _code(src.dtype), src.size, slab, n,
                       offsets, budget, out.ctypes.data, _code(out_dtype))
  return out


def check(src, slab, offsets, out_dtype, **kw):
  want = fake_ctx_reindex.gather(src, slab, offsets, out_dtype)
  np.testing.assert_array_equal(device_gather(src, slab, offsets, out_dtype),
                                want)
  np.testing.assert_array_equal(host_gather(src, slab, offsets, out_dtype,
                                            **kw), want)


@pytest.mark.parametrize('nlev', [13, 37])
@pytest.mark.parametrize('src_dtype,out_dtype', [
    (np.float32, np.float32), (np.float32, np.float64),
    (np.float64, np.float32), (np.float64, np.float64)])
def test_fullsize_slabs_every_dtype_pair_with_nan_slabs(nlev, src_dtype,
                                                        out_dtype):
  rs = np.random.RandomState(nlev)
  ntime = 3 if nlev == 13 else 2
  slab = nlev * GRID
  # realistic magnitudes (geopotential ~ 5e4) with float64 digits that
  # float32 must round
  src = (5e4 + 1e3 * rs.standard_normal(ntime * slab)).astype(src_dtype)
  offsets = np.array([slab, -1, 0, 2 * slab if ntime > 2 else slab, -1, 0])
  check(src, slab, offsets, out_dtype)


@pytest.mark.parametrize('slab', [4096, 4097, 4099, 70001, 1, 2, 3, 5, 1023,
                                  2048, 4095])
@pytest.mark.parametrize('dtypes', [(np.float32, np.float32),
                                    (np.float64, np.float32),
                                    (np.float32, np.float64)])
def test_misaligned_offsets_and_odd_slabs_on_both_kernels(slab, dtypes):
  rs = np.random.RandomState(slab)
  src = rs.standard_normal(40 * slab + 7).astype(dtypes[0])
  n = 257 if slab < 4096 else 13
  offsets = rs.randint(0, src.size - slab + 1, size=n)
  offsets[::5] = -1
  offsets[1] = src.size - slab  # the last valid offset
  check(src, slab, offsets, dtypes[1])


def test_slab_one_is_a_station_series():
  rs = np.random.RandomState(0)
  src = rs.standard_normal(100003).astype(np.float64)
  offsets = rs.randint(-1, src.size, size=300001)
  check(src, 1, offsets, np.float32)


def test_nothing_is_launched_for_nslab_or_slab_zero():
  import torch
  _lib, ctx = _ctx()
  x = torch.zeros(8, device='cuda')
  before = ctx.launch_count
  ctx.slab_gather(x.data_ptr(), _lib.F32, 8, 4, 0, np.zeros(0, np.int64), 0,
                  _lib.F32)
  ctx.slab_gather(x.data_ptr(), _lib.F32, 8, 0, 3, np.zeros(3, np.int64),
                  x.data_ptr(), _lib.F32)
  ctx.slab_gather_host(np.zeros(8, np.float32).ctypes.data, _lib.F32, 8, 4, 0,
                       np.zeros(0, np.int64), 1 << 20, 0, _lib.F32)
  assert ctx.launch_count == before


def test_invalid_tables_are_refused_on_the_host():
  import torch
  _lib, ctx = _ctx()
  x = torch.zeros(100, device='cuda')
  out = torch.zeros((2, 10), device='cuda')
  h = np.zeros(100, np.float32)
  ho = np.zeros((2, 10), np.float32)
  before = ctx.launch_count
  bad = [dict(offsets=[0, 91]), dict(offsets=[0, 2**62]),
         dict(src_elems=5, offsets=[-1, 0]), dict(src_dtype=2),
         dict(out_dtype=-1), dict(slab=-1), dict(nslab=-2)]
  for b in bad:
    kw = dict(src_dtype=_lib.F32, src_elems=100, slab=10, nslab=2,
              offsets=[0, 90], out_dtype=_lib.F32)
    kw.update(b)
    off = np.asarray(kw['offsets'], np.int64)
    with pytest.raises(_lib.Wb2Error):
      ctx.slab_gather(x.data_ptr(), kw['src_dtype'], kw['src_elems'],
                      kw['slab'], kw['nslab'], off, out.data_ptr(),
                      kw['out_dtype'])
    with pytest.raises(_lib.Wb2Error):
      ctx.slab_gather_host(h.ctypes.data, kw['src_dtype'], kw['src_elems'],
                           kw['slab'], kw['nslab'], off, 1 << 20,
                           ho.ctypes.data, kw['out_dtype'])
  with pytest.raises(_lib.Wb2Error, match='budget'):
    ctx.slab_gather_host(h.ctypes.data, _lib.F32, 100, 10, 2,
                         np.array([0, 90]), 8, ho.ctypes.data, _lib.F32)
  assert ctx.launch_count == before
  ctx.slab_gather(x.data_ptr(), _lib.F32, 100, 10, 2, np.array([0, 90]),
                  out.data_ptr(), _lib.F32)
  assert ctx.launch_count == before + 1


def test_memmap_source_uploads_only_the_referenced_slabs(tmp_path):
  _, ctx = _ctx()
  slab = 13 * 121 * 240
  mm = np.memmap(tmp_path / 'truth.f32', np.float32, 'w+', shape=(200, slab))
  mm[:] = np.arange(200, dtype=np.float32)[:, None] + np.linspace(0, 1, slab,
                                                                   dtype=np.float32)
  mm.flush()
  rs = np.random.RandomState(1)
  pos = rs.randint(0, 200, size=90)
  pos[:10] = pos[10]  # repeats
  pos[20:23] = [50, 51, 52]  # adjacent slabs: one copy
  pos[30] = -1
  offsets = np.where(pos < 0, -1, pos * slab)
  ctx.reset_transfer_stats()
  got = host_gather(mm, slab, offsets, np.float32)
  st = ctx.transfer_stats()
  referenced = np.unique(pos[pos >= 0]).size
  assert referenced < 90
  assert st['h2d_bytes'] == referenced * slab * 4
  assert st['d2h_bytes'] == 90 * slab * 4
  np.testing.assert_array_equal(got, fake_ctx_reindex.gather(
      np.asarray(mm).reshape(-1), slab, offsets, np.float32))


def test_small_budget_forces_many_bands_and_split_slabs():
  _, ctx = _ctx()
  rs = np.random.RandomState(2)
  for slab, budget in ((50021, 64 << 10), (50021, 1 << 20), (3, 1100),
                       (4096, 9000)):
    src = rs.standard_normal(20 * slab + 3).astype(np.float64)
    offsets = rs.randint(-1, src.size - slab + 1, size=17)
    before = ctx.launch_count
    want = fake_ctx_reindex.gather(src, slab, offsets, np.float32)
    np.testing.assert_array_equal(
        host_gather(src, slab, offsets, np.float32, budget=budget), want)
    assert ctx.launch_count - before >= 4, (slab, budget)


# -- the three operations end to end ------------------------------------------
def _to_device(ds):
  import torch
  from weatherbench2_b200 import xarray_lite as xl
  out = xl.Dataset(coords=ds.coords, attrs=ds.attrs)
  for k, v in ds.items():
    out[k] = xl.DataArray(torch.from_numpy(np.ascontiguousarray(v.values)).cuda(),
                          v.dims, v.coords, k, v.attrs)
  return out


def _all_cuda(out):
  import torch
  for name, da in out.items():
    if name != 'source_time':
      assert isinstance(da.data, torch.Tensor) and da.data.is_cuda, name


@pytest.mark.parametrize('dims', IVT_DIMS, ids=lambda d: '-'.join(d))
@pytest.mark.parametrize('mode', ['valid_and_delta', 'valid_and_init'])
def test_index_on_valid_time_on_the_gpu(dims, mode):
  ivt_case(dims, mode, np.float64, 3, ncell=GRID // 1440 * 8)
  _all_cuda(ivt_case(dims, mode, np.float32, 4, ncell=1440,
                     to_device=_to_device))
  ivt_case(dims, mode, np.int32, 5, to_device=_to_device)


@pytest.mark.parametrize('dims', CLIM_DIMS, ids=lambda d: '-'.join(d))
def test_expand_climatology_on_the_gpu(dims):
  expand_case(dims, '2019-12-01', '2020-03-30')
  _all_cuda(expand_case(dims, '2020-02-20', '2020-03-10', np.float64,
                        to_device=_to_device))


@pytest.mark.parametrize('dims', TRUTH_DIMS, ids=lambda d: '-'.join(d))
def test_probabilistic_forecasts_on_the_gpu(dims, monkeypatch):
  prob_case(dims)
  _all_cuda(prob_case(dims, to_device=_to_device, dtype=np.float64))
  from weatherbench2_b200 import reindexing
  monkeypatch.setattr(reindexing, 'STREAM_BUDGET_BYTES', 4 << 10)
  prob_case(dims, initial_time_end='1991-01-02')

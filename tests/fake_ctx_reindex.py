"""TEST INFRASTRUCTURE: NumPy interpretation of wb2_slab_gather /
wb2_slab_gather_host (include/wb2b200.h) on top of `fake_ctx.FakeContext`, so
that weatherbench2_b200.reindexing runs end to end on a CPU.  It reads the
source and the offset table the operators hand to the library, checks the
table as the C entry does, and copies slab by slab (the kernels' vector and
flat paths and the host entry's bands are checked by the GPU tests)."""
import numpy as np

import fake_ctx
from fake_ctx import _view
from weatherbench2_b200 import _lib


def gather(src: np.ndarray, slab: int, offsets, out_dtype) -> np.ndarray:
  """out[s] = src[offsets[s]:offsets[s] + slab] cast to out_dtype, or NaN
  where offsets[s] < 0; raises Wb2Error for a table the C entry refuses."""
  off = np.asarray(offsets, np.int64).reshape(-1)
  ok = off >= 0
  if ok.any() and (slab > src.size or off[ok].max() > src.size - slab):
    raise _lib.Wb2Error('wb2_slab_gather: a slab ends past src_elems')
  out = np.full((off.size, slab), np.nan, out_dtype)
  if slab <= 64:
    out[ok] = src[off[ok, None] + np.arange(slab)[None, :]].astype(out_dtype)
  else:
    for s in np.flatnonzero(ok):
      out[s] = src[off[s]:off[s] + slab]
  return out


class ReindexFakeContext(fake_ctx.FakeContext):
  """FakeContext plus the slab gather entries."""

  def slab_gather(self, src, src_dtype, src_elems, slab, nslab, offsets, out,
                  out_dtype=_lib.F32):
    self.calls.append(('slab_gather', int(nslab), int(slab)))
    self._run(src, src_dtype, src_elems, slab, nslab, offsets, out, out_dtype)

  def slab_gather_host(self, src, src_dtype, src_elems, slab, nslab, offsets,
                       budget, out, out_dtype=_lib.F32):
    self.calls.append(('slab_gather_host', int(nslab), int(slab), int(budget)))
    self._run(src, src_dtype, src_elems, slab, nslab, offsets, out, out_dtype)

  @staticmethod
  def _run(src, src_dtype, src_elems, slab, nslab, offsets, out, out_dtype):
    assert np.asarray(offsets).size == nslab
    ti = np.float32 if src_dtype == _lib.F32 else np.float64
    to = np.float32 if out_dtype == _lib.F32 else np.float64
    res = gather(_view(src, int(src_elems), ti), int(slab), offsets, to)
    _view(out, res.size, to)[...] = res.reshape(-1)


def installed():
  """Makes `_lib.default_context()` return a ReindexFakeContext."""
  return fake_ctx.installed(ReindexFakeContext)

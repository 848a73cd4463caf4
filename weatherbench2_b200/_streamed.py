"""Where the data of a streamed operator lives decides which C entry runs it.

The quantile, average, time-window, precipitation-accumulation and
climatology operators each have an entry pair in `_lib.Context`:
`X(x, dtype, *args, *outputs)` reads device addresses, and
`X_host(x, dtype, *args, budget, *outputs)` streams host memory through the
device in bands whose device footprint stays within `budget` bytes.  `run`
holds the one rule that picks between them, so each operator only computes
its layout."""
from __future__ import annotations

import functools
import math
from typing import Optional, Sequence

import numpy as np

from weatherbench2_b200 import _lib
from weatherbench2_b200 import xarray_lite as xl


@functools.lru_cache(maxsize=None)
def _torch_dtype(dtype):
  """torch.float32 for np.float32 and so on (cached: `np.dtype.name` takes
  microseconds, as long as the rest of a small call)."""
  import torch  # pylint: disable=import-outside-toplevel
  return getattr(torch, np.dtype(dtype).name)


def run(entry: str, data, args: Sequence, outputs: Sequence, budget: int, *,
        perm: Optional[Sequence[int]] = None, dtype=None, **kwargs) -> list:
  """Runs `entry` of the default context on `data` (a variable's `.data`)
  and returns its outputs in order.

  A CUDA tensor stays on its device: it is permuted by `perm`, cast to
  `dtype` and made contiguous, its outputs are `torch.empty` on that device,
  and `entry` runs on device addresses.  Anything else is read as NumPy (as
  `DataArray.values` does), transposed by `perm` and made contiguous in
  `dtype`; its outputs come from the context's pinned pool, and
  `entry + '_host'` streams it through the device within `budget` bytes.
  Data already contiguous in the layout and dtype asked for is read in place,
  without a copy.

  `perm` None keeps the stored order and `dtype` None the stored dtype.  The
  dtype after the cast gives the entry's dtype code (float64: WB2_F64, any
  other: WB2_F32), so callers accept only float32 and float64.  `outputs` lists one (shape, NumPy dtype) per output of the entry, or
  None for an output not asked for, which the entry gets as a NULL pointer
  and which is returned as None.  `kwargs` go to the entry as they are.
  When every output asked for is empty the entry is not called."""
  ctx = _lib.default_context()
  if xl._is_torch(data) and data.is_cuda:  # pylint: disable=protected-access
    import torch  # pylint: disable=import-outside-toplevel
    x = data if perm is None else data.permute(*perm)
    x = (x if dtype is None else x.to(_torch_dtype(dtype))).contiguous()
    code = _lib.F64 if x.dtype == torch.float64 else _lib.F32
    res = [None if o is None else
           torch.empty(o[0], dtype=_torch_dtype(o[1]), device=x.device)
           for o in outputs]
    fn, extra, ptr = getattr(ctx, entry), (), lambda a: a.data_ptr()
  else:
    x = xl._np(data)  # pylint: disable=protected-access
    x = np.ascontiguousarray(x if perm is None else np.transpose(x, perm),
                             dtype=dtype)
    code = _lib.F64 if x.dtype == np.float64 else _lib.F32
    res = [None if o is None else ctx.pinned_result(*o) for o in outputs]
    fn, extra, ptr = (getattr(ctx, entry + '_host'), (budget,),
                      lambda a: a.ctypes.data)
  if any(math.prod(o[0]) for o in outputs if o is not None):
    fn(ptr(x), code, *args, *extra,
       *[None if a is None else ptr(a) for a in res], **kwargs)
  return res

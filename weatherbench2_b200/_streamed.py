"""Where an operator's data lives decides how its C entry runs: the one
residency rule of the operators, in two forms.

`place` serves the operators with an entry pair in `_lib.Context`, a device
entry and a `_host` twin that streams host memory through the device: the
zonal spectrum and the conservative regridder directly, and the quantile,
average, time-window, precipitation-accumulation and climatology operators
through `run`.  The derived-variable, ensemble-mean, spectrum-interpolation
and nearest and bilinear regrid operators have only the device entry:
`run_whole` runs it on CUDA operands in place, and otherwise uploads the host
operands whole and copies the results back.  Either way each operator only
computes its layout."""
from __future__ import annotations

import functools
import math
from typing import Optional, Sequence

import numpy as np

from weatherbench2_b200 import _lib
from weatherbench2_b200 import _spatial
from weatherbench2_b200 import xarray_lite as xl


@functools.lru_cache(maxsize=None)
def _torch_dtype(dtype):
  """torch.float32 for np.float32 and so on (cached: `np.dtype.name` takes
  microseconds, as long as the rest of a small call)."""
  import torch  # pylint: disable=import-outside-toplevel
  return getattr(torch, np.dtype(dtype).name)


def place(data, outputs: Sequence, device, host, *,
          perm: Optional[Sequence[int]] = None, dtype=None) -> list:
  """The placement half of `run`, for any entry pair: lays out `data` (a
  variable's `.data`) and allocates the outputs as `run` describes, runs
  `device(x, code, *outs)` on a CUDA tensor and `host(x, code, *outs)` on
  anything else, and returns the outputs in order.  `code` is the entry's
  dtype code of `x`.  The arms get arrays rather than addresses, so that a
  device arm can initialise an output on torch's current stream; an output
  not asked for is None.  When every output asked for is empty no arm runs."""
  if xl._is_torch(data) and data.is_cuda:  # pylint: disable=protected-access
    import torch  # pylint: disable=import-outside-toplevel
    x = data if perm is None else data.permute(*perm)
    x = (x if dtype is None else x.to(_torch_dtype(dtype))).contiguous()
    code = _lib.F64 if x.dtype == torch.float64 else _lib.F32
    res = [None if o is None else
           torch.empty(o[0], dtype=_torch_dtype(o[1]), device=x.device)
           for o in outputs]
    arm = device
  else:
    x = xl._np(data)  # pylint: disable=protected-access
    x = np.ascontiguousarray(x if perm is None else np.transpose(x, perm),
                             dtype=dtype)
    code = _lib.F64 if x.dtype == np.float64 else _lib.F32
    ctx = _lib.default_context()
    res = [None if o is None else ctx.pinned_result(*o) for o in outputs]
    arm = host
  if any(math.prod(o[0]) for o in outputs if o is not None):
    arm(x, code, *res)
  return res


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

  def device(x, code, *res):
    getattr(ctx, entry)(x.data_ptr(), code, *args, *[
        None if a is None else a.data_ptr() for a in res], **kwargs)

  def host(x, code, *res):
    getattr(ctx, entry + '_host')(x.ctypes.data, code, *args, budget, *[
        None if a is None else a.ctypes.data for a in res], **kwargs)

  return place(data, outputs, device, host, perm=perm, dtype=dtype)


def run_whole(datas: Sequence, outputs: Sequence, call, *,
              perms: Optional[Sequence] = None, dtype=None) -> list:
  """Runs `call(in_ptrs, out_ptrs)` once on device copies of `datas` (the
  operands' `.data`) and returns its outputs in order.

  When any operand is a CUDA tensor the call runs on that tensor's device:
  every operand is moved there (NumPy through `torch.from_numpy`), permuted by
  its entry of `perms`, cast to `dtype` and made contiguous, and the outputs
  are `torch.empty` on that device.  Otherwise every operand is read as NumPy,
  transposed and made contiguous in `dtype`, uploaded whole, and the outputs
  come back as NumPy; every device buffer is freed when the call returns or
  raises.  `perms` None, or a None entry, keeps the stored order, and `dtype`
  None the stored dtype.  `outputs` lists one (shape, NumPy dtype) per output.
  When every output is empty, `call` is not made and nothing is uploaded."""
  perms = [None] * len(datas) if perms is None else perms
  empty = not any(math.prod(shape) for shape, _ in outputs)
  device = next((x.device for x in datas
                 if xl._is_torch(x) and x.is_cuda), None)  # pylint: disable=protected-access
  if device is not None:
    import torch  # pylint: disable=import-outside-toplevel
    res = [torch.empty(shape, dtype=_torch_dtype(dt), device=device)
           for shape, dt in outputs]
    if empty:
      return res
    xs = []
    for x, perm in zip(datas, perms):
      if not xl._is_torch(x):  # pylint: disable=protected-access
        x = torch.from_numpy(xl._np(x))  # pylint: disable=protected-access
      if perm is not None:
        x = x.permute(*perm)
      xs.append(x.to(device, None if dtype is None else _torch_dtype(dtype))
                .contiguous())
    # No host wait: _LockedLib orders the entry after torch's current stream
    # and that stream after the entry, so torch may reuse `xs` once freed.
    call([x.data_ptr() for x in xs], [r.data_ptr() for r in res])
    return res
  if empty:
    return [np.empty(shape, dt) for shape, dt in outputs]
  xs = [np.ascontiguousarray(
      xl._np(x) if perm is None else np.transpose(xl._np(x), perm),  # pylint: disable=protected-access
      dtype=dtype) for x, perm in zip(datas, perms)]
  ctx = _lib.default_context()
  with _spatial.Staging(ctx) as stage:
    ins = [stage.array(x) for x in xs]
    outs = [stage.malloc(math.prod(shape) * np.dtype(dt).itemsize)
            for shape, dt in outputs]
    call(ins, outs)
    return [ctx.from_device(p, shape, dt)
            for p, (shape, dt) in zip(outs, outputs)]

"""Device-side preprocessing that feeds the metric kernels (SURVEY.md section 8
f3): the ensemble mean of scripts/compute_ensemble_mean.py:110-141
(`xbeam.Mean(realization, skipna)`) computed in HBM, so that ensemble-mean
RMSE / ACC through K1 need no host round trip of the mean; and the quantiles
of scripts/compute_quantiles.py (`Dataset.quantile` over chosen dims,
csrc/quantile.cu)."""
from __future__ import annotations

import math
from typing import Optional, Sequence

import numpy as np
import pandas as pd

from weatherbench2_b200 import _lib
from weatherbench2_b200 import xarray_lite as xl

REALIZATION = 'realization'
QUANTILE = 'quantile'
# device bytes of the two staging buffers of a host (NumPy) quantile call
QUANTILE_STREAM_BUDGET_BYTES = 1 << 30


def compute_ensemble_mean(dataset, realization_name: str = REALIZATION,
                          skipna: bool = False):
  """Mean over `realization_name` of every variable that has it
  (scripts/compute_ensemble_mean.py:131: xbeam.Mean(REALIZATION_NAME, skipna)).

  float32 like xarray's mean of float32 data.  CUDA-tensor variables stay on
  the device (the result is a CUDA tensor K1 / K6 read in place); NumPy
  variables are uploaded, reduced and the (M times smaller) mean comes back.
  Variables without the dimension pass through.
  """
  native = xl.is_native_xarray(dataset)
  ds = xl.from_xarray(dataset)
  ctx = _lib.default_context()
  out = xl.Dataset(attrs=ds.attrs)
  for name in ds.keys():
    v = ds[name]
    if realization_name not in v.dims:
      out[name] = v
      continue
    dims = tuple(d for d in v.dims if d != realization_name)
    work = v.transpose(realization_name, *dims)
    data = work.data
    m = work.sizes[realization_name]
    shape = tuple(work.sizes[d] for d in dims)
    cells = int(np.prod(shape)) if shape else 1
    # one flat "field" per variable: the kernel walks it with a 64-bit
    # grid-stride loop, members `cells` elements apart
    slab = cells
    off = np.zeros(1, dtype=np.int64)
    coords = {k: c for k, c in work.coords.items()
              if realization_name not in c.dims}
    if xl._is_torch(data) and data.is_cuda:  # pylint: disable=protected-access
      import torch  # pylint: disable=import-outside-toplevel
      x = data.to(torch.float32).contiguous()
      res = torch.empty(shape, device=x.device, dtype=torch.float32)
      ctx.ens_mean(x.data_ptr(), m, cells, off, slab, skipna, res.data_ptr())
      values = res
    else:
      x = np.ascontiguousarray(np.asarray(data), dtype=np.float32)
      src = ctx.to_device(x)
      dst = ctx.malloc(max(4, cells * 4))
      try:
        ctx.ens_mean(src, m, cells, off, slab, skipna, dst)
        values = ctx.from_device(dst, shape, np.float32)
      finally:
        ctx.free(src)
        ctx.free(dst)
    out[name] = xl.DataArray(values, dims, coords, name, v.attrs)
  return xl.to_xarray(out) if native else out


def _check_quantiles(quantiles) -> list:
  quantiles = [float(q) for q in quantiles]
  if any(not 0 <= q <= 1 for q in quantiles):  # NaN fails both comparisons
    raise ValueError(
        f'Expected all quantiles to be in [0, 1]. Found {quantiles=}')
  if not quantiles or len(quantiles) > _lib.MAX_QUANTILES:
    raise ValueError(f'between 1 and {_lib.MAX_QUANTILES} quantiles are '
                     f'supported per call (got {len(quantiles)})')
  return quantiles


def _variable_quantiles(v: xl.DataArray, reduce: list, quantiles: list,
                        skipna: bool):
  """The quantiles of `v` over the dims `reduce`: [nq, *preserved shape], a
  CUDA tensor for CUDA data, else NumPy.  Adjacent reduced dims are read in
  place as [outer][n][inner]; otherwise one transposed contiguous copy with
  the reduced dims in front is made first (torch on the device, NumPy on the
  host)."""
  if v.dtype not in (np.float32, np.float64):
    raise TypeError(f'variable {v.name!r} has dtype {v.dtype}: quantiles '
                    'take float32 or float64 data')
  pos = sorted(v.dims.index(d) for d in reduce)
  keep = [d for d in v.dims if d not in reduce]
  nsample = math.prod(v.sizes[d] for d in reduce)
  if nsample == 0:
    raise ValueError(f'variable {v.name!r}: cannot take quantiles over an '
                     f'empty reduction ({reduce})')
  perm = None
  if not pos:  # a 0-d variable: one sample
    nouter = ninner = 1
  elif pos[-1] - pos[0] == len(pos) - 1:
    nouter = math.prod(v.shape[:pos[0]])
    ninner = math.prod(v.shape[pos[-1] + 1:])
  else:
    nouter, ninner = 1, math.prod(v.sizes[d] for d in keep)
    perm = pos + [v.dims.index(d) for d in keep]
  code = _lib.F64 if v.dtype == np.float64 else _lib.F32
  nq = len(quantiles)
  out_shape = (nq,) + tuple(v.sizes[d] for d in keep)
  ctx = _lib.default_context()
  data = v.data
  if xl._is_torch(data) and data.is_cuda:  # pylint: disable=protected-access
    import torch  # pylint: disable=import-outside-toplevel
    x = (data if perm is None else data.permute(*perm)).contiguous()
    out = torch.empty(out_shape, dtype=torch.float64, device=x.device)
    if out.numel():
      ctx.quantile(x.data_ptr(), code, nouter, nsample, ninner, quantiles,
                   skipna, out.data_ptr())
    return out
  x = np.asarray(data)
  x = np.ascontiguousarray(x if perm is None else np.transpose(x, perm))
  out = ctx.pinned_result(out_shape, np.float64)
  if out.size:
    ctx.quantile_host(x.ctypes.data, code, nouter, nsample, ninner, quantiles,
                      skipna, QUANTILE_STREAM_BUDGET_BYTES, out.ctypes.data)
  return out


def compute_quantiles_core(chunk, quantiles: Sequence[float], dim, *,
                           skipna: bool = False, name_suffix: str = ''):
  """`_evaluate_chunk_core` of scripts/compute_quantiles.py:168-183:
  `chunk.quantile(quantiles, dim=dim, skipna=skipna)` (method 'linear') with
  every variable `v` renamed `v + name_suffix`.

  Like xarray's Dataset.quantile: a float64 `quantile` dimension comes first,
  then the preserved dims in input order; coordinates along reduced dims are
  dropped; a variable with none of the reduced dims passes through; attrs
  are dropped.  The values are numpy's np.quantile / np.nanquantile bit for
  bit, as float64 (include/wb2b200.h, DESIGN.md section 8f).  CUDA-tensor
  variables give CUDA tensors; NumPy or memmap variables are streamed
  through the device in bands and give NumPy.  Reduced dims need not be
  adjacent: when they are not, the variable is copied once, transposed with
  the reduced dims in front (torch on the device, NumPy on the host)."""
  native = xl.is_native_xarray(chunk)
  ds = xl.from_xarray(chunk)
  dims = [dim] if isinstance(dim, str) else list(dim)
  preserve_dims = set(d for d in ds.dims if d not in dims)
  if not preserve_dims.issubset(set(ds.dims)):
    raise ValueError(
        f'User specified dim={dims}, which results in preserved dims'
        f' {preserve_dims} , not being a subset of {set(ds.dims)=}')
  quantiles = _check_quantiles(quantiles)
  missing = [d for d in dims if d not in ds.dims]
  if missing:
    raise ValueError(f'Dimensions {tuple(missing)} not found in data '
                     f'dimensions {tuple(ds.dims)}')
  coords = {k: c for k, c in ds.coords.items()
            if not any(d in dims for d in c.dims)}
  coords[QUANTILE] = xl.Coord((QUANTILE,), np.asarray(quantiles, np.float64))
  out = xl.Dataset(coords=coords)
  for name in ds.keys():
    v = ds[name]
    reduce = [d for d in v.dims if d in dims]
    if not reduce and v.dims:
      out[name + name_suffix] = xl.DataArray(v.data, v.dims, attrs=v.attrs)
      continue
    values = _variable_quantiles(v, reduce, quantiles, skipna)
    out[name + name_suffix] = xl.DataArray(
        values, (QUANTILE,) + tuple(d for d in v.dims if d not in reduce))
  return xl.to_xarray(out) if native else out


def compute_quantiles(ds, quantiles: Sequence[float], dim, *,
                      skipna: bool = False, name_suffix: str = '',
                      variables: Optional[Sequence[str]] = None,
                      levels: Optional[Sequence] = None,
                      time_dim: str = 'time',
                      time_start: Optional[str] = '2020-01-01',
                      time_stop: Optional[str] = '2020-12-31'):
  """scripts/compute_quantiles.py `main` without Beam or zarr: the script's
  `_impose_data_selection` (variables, then [time_start, time_stop] on
  `time_dim` with both ends inclusive and the script's default range, then
  `levels` on `level`, each only where the dim exists), then
  `compute_quantiles_core`."""
  native = xl.is_native_xarray(ds)
  ds = xl.from_xarray(ds)
  if variables is not None:
    ds = ds[list(variables)]
  if time_dim in ds.dims:
    index = pd.Index(ds.coords[time_dim].values)
    ds = ds.isel({time_dim: index.slice_indexer(time_start, time_stop)})
  if levels and 'level' in ds.dims:
    ds = ds.sel(level=[float(l) for l in levels])
  out = compute_quantiles_core(ds, quantiles, dim, skipna=skipna,
                               name_suffix=name_suffix)
  return xl.to_xarray(out) if native else out

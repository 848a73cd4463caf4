"""Host-side planning for the spatial-reduction kernels.

Turns named-dimension arrays (NumPy on the host or torch tensors on a CUDA
device) plus a list of regions into what the C ABI wants: a base pointer and a
per-field element-offset table for every operand, and a `wb2_weights`
description of latitude weights x region masks.  Nothing numerical happens
here except building the (tiny) weight vectors with the reference's own
formulas (weatherbench2/metrics.py:35-60).
"""
from __future__ import annotations

import dataclasses
from typing import Optional, Sequence

import numpy as np

from weatherbench2_b200 import _lib
from weatherbench2_b200 import xarray_lite as xl

LAT, LON = 'latitude', 'longitude'


# ---- latitude weights (metrics.py:35-60) -------------------------------------
def _assert_increasing(x: np.ndarray):
  if not (np.diff(x) > 0).all():
    raise ValueError(f'array is not increasing: {x}')


def _latitude_cell_bounds(x: np.ndarray) -> np.ndarray:
  pi_over_2 = np.array([np.pi / 2], dtype=x.dtype)
  return np.concatenate([-pi_over_2, (x[:-1] + x[1:]) / 2, pi_over_2])


def _cell_area_from_latitude(points: np.ndarray) -> np.ndarray:
  bounds = _latitude_cell_bounds(points)
  _assert_increasing(bounds)
  return np.sin(bounds[1:]) - np.sin(bounds[:-1])


def lat_weights(latitude_deg: np.ndarray) -> np.ndarray:
  """Area weights normalised to mean 1 (weatherbench2/metrics.py:55-60)."""
  w = _cell_area_from_latitude(np.deg2rad(np.asarray(latitude_deg)))
  return w / np.mean(w)


# ---- operand description -----------------------------------------------------
@dataclasses.dataclass
class Operand:
  """One named array prepared for the kernels."""
  data: object               # np.ndarray or torch.Tensor (kept alive)
  addr: int                  # address of element 0
  itemsize: int
  on_device: bool
  outer_dims: tuple          # non-spatial dims
  outer_shape: tuple
  outer_strides: tuple       # in elements
  layout: str                # 'lat_lon' (lon contiguous) | 'lon_lat'
  nrow: int
  ncol: int
  row_stride: int
  dtype: np.dtype


def _strides_elems(data) -> tuple:
  if xl._is_torch(data):  # pylint: disable=protected-access
    return tuple(int(s) for s in data.stride())
  return tuple(int(s // data.itemsize) for s in data.strides)


def _address(data) -> int:
  if xl._is_torch(data):  # pylint: disable=protected-access
    return int(data.data_ptr())
  return int(data.ctypes.data)


def _np_dtype(data) -> np.dtype:
  if xl._is_torch(data):  # pylint: disable=protected-access
    return np.dtype(str(data.dtype).replace('torch.', ''))
  return data.dtype


def prepare_operand(da: xl.DataArray, want_layout: Optional[str] = None,
                    want_dtype: Optional[np.dtype] = None) -> Operand:
  """Describes `da` for the kernels, copying only when its memory layout is
  not (…outer…, row, col) with `col` contiguous, or its dtype is neither
  float32 nor float64."""
  if LAT not in da.dims or LON not in da.dims:
    raise ValueError(f'{da.name!r} needs latitude and longitude dims, has '
                     f'{da.dims}')
  lazy = getattr(da, 'lazy_source', None)
  if lazy is not None:
    # a label gather (e.g. truth.sel(time=valid_time)): address the source
    # through the offset table instead of materialising the copy
    source, maps = lazy
    return gather_operand(prepare_operand(source, want_layout, want_dtype),
                          maps)
  data = da.data
  dims = da.dims
  torch_in = xl._is_torch(data)  # pylint: disable=protected-access
  dt = _np_dtype(data)
  target_dt = np.dtype(want_dtype) if want_dtype is not None else (
      dt if dt in (np.dtype('float32'), np.dtype('float64'))
      else np.dtype('float32') if dt.itemsize <= 4 and dt.kind == 'f'
      else np.dtype('float64'))
  if dt != target_dt:
    if torch_in:
      import torch  # pylint: disable=import-outside-toplevel
      data = data.to(getattr(torch, target_dt.name))
    else:
      data = data.astype(target_dt)
  strides = _strides_elems(data)
  ilat, ilon = dims.index(LAT), dims.index(LON)
  shape = tuple(data.shape)

  def slab_is_whole(irow, icol):
    # no other dimension may be interleaved with the (row, col) slab: every
    # outer stride spans a whole slab (or is 0: a broadcast view).  Otherwise
    # the slab of one field is scattered through memory -- two operands with
    # the same dims in a different order would disagree on the row stride, and
    # the kernels would stride through HBM -- so such arrays are compacted.
    span = (shape[irow] - 1) * strides[irow] + shape[icol]
    return all(shape[i] == 1 or strides[i] == 0 or strides[i] >= span
               for i in range(len(shape)) if i not in (irow, icol))

  def layout_ok():
    # rows must also be densely packed (row stride == ncol): operands of one
    # launch share ONE row stride in the C ABI, and a strided view on one side
    # (a longitude box, every second row, an integer pick of an inner
    # dimension) against a dense array on the other would otherwise be
    # refused.  Such views are compacted; whole-slab views stay zero-copy.
    if strides[ilon] == 1 or shape[ilon] == 1:
      lay = 'lat_lon'
      if (strides[ilat] == shape[ilon] or shape[ilat] == 1) and slab_is_whole(
          ilat, ilon):
        return lay
    if strides[ilat] == 1 or shape[ilat] == 1:
      lay = 'lon_lat'
      if (strides[ilon] == shape[ilat] or shape[ilon] == 1) and slab_is_whole(
          ilon, ilat):
        return lay
    return None

  lay = layout_ok()
  if any(s < 0 for s in strides):
    lay = None
  if lay is None or (want_layout is not None and lay != want_layout and not (
      shape[ilat] == 1 or shape[ilon] == 1)):
    # contiguous copy with the spatial dims last, in the wanted order
    order = want_layout or 'lat_lon'
    sp = (LAT, LON) if order == 'lat_lon' else (LON, LAT)
    perm_dims = tuple(d for d in dims if d not in sp) + sp
    perm = [dims.index(d) for d in perm_dims]
    if torch_in:
      data = data.permute(*perm).contiguous()
    else:
      data = np.ascontiguousarray(np.transpose(data, perm))
    dims = perm_dims
    strides = _strides_elems(data)
    shape = tuple(data.shape)
    ilat, ilon = dims.index(LAT), dims.index(LON)
    lay = order
  if want_layout is not None and lay != want_layout:
    lay = want_layout  # degenerate size-1 axis: either description is valid
  if lay == 'lat_lon':
    nrow, ncol, row_stride = shape[ilat], shape[ilon], strides[ilat]
  else:
    nrow, ncol, row_stride = shape[ilon], shape[ilat], strides[ilon]
  if nrow == 1:
    row_stride = max(row_stride, ncol)
  outer = [i for i in range(len(dims)) if i not in (ilat, ilon)]
  on_dev = bool(torch_in and data.is_cuda)
  if torch_in and not on_dev:
    data = data.numpy()
  return Operand(
      data=data, addr=_address(data), itemsize=target_dt.itemsize,
      on_device=on_dev, outer_dims=tuple(dims[i] for i in outer),
      outer_shape=tuple(shape[i] for i in outer),
      outer_strides=tuple(strides[i] for i in outer), layout=lay, nrow=nrow,
      ncol=ncol, row_stride=int(row_stride), dtype=target_dt)


def broadcast_dims(*operands: Operand) -> tuple[tuple, tuple]:
  """Result dims/shape of xarray arithmetic between the operands: dims of the
  first, then unseen dims of the next ones."""
  dims, shape = [], []
  for op in operands:
    for d, n in zip(op.outer_dims, op.outer_shape):
      if d in dims:
        if shape[dims.index(d)] != n:
          raise ValueError(
              f'size mismatch along {d!r}: {shape[dims.index(d)]} vs {n}')
      else:
        dims.append(d)
        shape.append(n)
  return tuple(dims), tuple(shape)


def offset_table(op: Operand, dims: tuple, shape: tuple) -> np.ndarray:
  """Element offset of the slab of `op` for every index of the broadcast outer
  grid (C order).  Missing dims get stride 0 (broadcast)."""
  off = np.zeros(shape, dtype=np.int64)
  gathered = getattr(op, 'gather_terms', None)
  if gathered is not None:
    # explicit (dims, offsets) terms: a label lookup folded into the table
    for tdims, arr in gathered:
      perm = [tdims.index(d) for d in dims if d in tdims]
      a = np.transpose(np.asarray(arr, dtype=np.int64), perm)
      a = a[tuple(slice(None) if d in tdims else None for d in dims)]
      off = off + a
    return np.ascontiguousarray(np.broadcast_to(off, shape)).reshape(-1)
  for ax, (d, n) in enumerate(zip(dims, shape)):
    if d in op.outer_dims:
      st = op.outer_strides[op.outer_dims.index(d)]
      sh = [1] * len(shape)
      sh[ax] = n
      off = off + (np.arange(n, dtype=np.int64) * st).reshape(sh)
  return np.ascontiguousarray(off).reshape(-1)


def gather_operand(op: Operand, index_maps: dict) -> Operand:
  """Re-addresses `op` through label lookups without copying data.

  index_maps: {source_dim: (new_dims, positions)} -- `source_dim` of `op` is
  indexed by the integer array `positions` whose dims are `new_dims`
  (xarray's vectorised `.sel`, e.g. the day-of-year / hour lookup of
  weatherbench2/metrics.py:398-404 or `truth.sel(time=valid_time)`,
  evaluation.py:475).  Untouched outer dims keep their stride addressing.
  """
  terms = []
  new_dims, new_shape = [], []

  def add_dim(d, n):
    if d in new_dims:
      if new_shape[new_dims.index(d)] != n:
        raise ValueError(f'size mismatch along {d!r}')
    else:
      new_dims.append(d)
      new_shape.append(n)

  for d, n, st in zip(op.outer_dims, op.outer_shape, op.outer_strides):
    if d in index_maps:
      tdims, pos = index_maps[d]
      pos = np.asarray(pos, dtype=np.int64)
      if pos.size and (pos.min() < 0 or pos.max() >= n):
        raise IndexError(f'gather positions out of range for {d!r}')
      terms.append((tuple(tdims), pos * st))
      for td, tn in zip(tdims, pos.shape):
        add_dim(td, tn)
    else:
      terms.append(((d,), np.arange(n, dtype=np.int64) * st))
      add_dim(d, n)
  out = dataclasses.replace(op, outer_dims=tuple(new_dims),
                            outer_shape=tuple(new_shape),
                            outer_strides=tuple(0 for _ in new_dims))
  out.gather_terms = terms
  return out


# ---- weights -----------------------------------------------------------------
def region_factors(regions: Sequence, latitude: np.ndarray,
                   longitude: np.ndarray):
  out = []
  for r in regions:
    if r is None:
      from weatherbench2_b200.regions import RegionFactors  # pylint: disable=import-outside-toplevel
      out.append(RegionFactors(np.ones(latitude.size), np.ones(longitude.size)))
    else:
      out.append(r.factors(latitude, longitude))
  return out


def _segments(factors_along_col: np.ndarray):
  """Column segments on which every region's factor is constant.
  factors_along_col: [R, ncol].  Returns (seg_start[nseg+1], seg_w[R, nseg])."""
  ncol = factors_along_col.shape[1]
  change = np.any(factors_along_col[:, 1:] != factors_along_col[:, :-1], axis=0)
  starts = np.concatenate([[0], np.nonzero(change)[0] + 1]).astype(np.int32)
  seg_start = np.concatenate([starts, [ncol]]).astype(np.int32)
  seg_w = factors_along_col[:, starts]
  return seg_start, np.ascontiguousarray(seg_w, dtype=np.float64)


def build_weights(ctx: _lib.Context, latitude: np.ndarray,
                  longitude: np.ndarray, regions: Sequence, layout: str,
                  row_stride: int, cell_cache: Optional[dict] = None,
                  max_regions: int = _lib.MAX_REGIONS
                  ) -> list[tuple[list[int], _lib.WeightSpec]]:
  """WeightSpecs for `regions` (entries may be None = global).

  Regions that carry a 2-D mask (LandRegion) cannot share a launch with a
  different mask, so the result is a list of (region indices, WeightSpec)
  groups; regions without a mask all go in the first group.
  """
  wlat = lat_weights(latitude)
  facs = region_factors(regions, latitude, longitude)
  if cell_cache is not None:
    # the cached values are DEVICE pointers: they belong to this context (its
    # device, its lifetime), whatever dict the caller passed to ask for caching
    cell_cache = ctx.__dict__.setdefault('_cell_weight_cache', {})
  groups: dict = {}
  for i, fc in enumerate(facs):
    key = None if fc.cell is None else fc.cell.tobytes()
    groups.setdefault(key, []).append(i)
  out = []
  nlat, nlon = latitude.size, longitude.size
  for key, idx in groups.items():
    for j0 in range(0, len(idx), max_regions):
      ids = idx[j0:j0 + max_regions]
      latf = np.stack([facs[i].lat for i in ids])  # [R, nlat]
      lonf = np.stack([facs[i].lon for i in ids])  # [R, nlon]
      zero_skip = any(regions[i] is not None for i in ids)
      cell_dev = None
      if key is not None:
        cell = facs[ids[0]].cell
        cell = cell if layout == 'lat_lon' else cell.T
        cache_key = (key, cell.shape, layout)
        if cell_cache is not None and cache_key in cell_cache:
          cell_dev = cell_cache[cache_key]
        else:
          cell_dev = ctx.to_device(np.ascontiguousarray(cell, np.float32))
          if cell_cache is not None:
            cell_cache[cache_key] = cell_dev
      if layout == 'lat_lon':
        seg_start, seg_w = _segments(lonf)
        spec = _lib.WeightSpec(nlat, nlon, latf * wlat[None, :], seg_start,
                               seg_w, None, cell_dev, zero_skip, row_stride)
      else:
        seg_start, seg_w = _segments(latf)
        spec = _lib.WeightSpec(nlon, nlat, lonf, seg_start, seg_w,
                               wlat.astype(np.float32), cell_dev, zero_skip,
                               row_stride)
      out.append((ids, spec))
  return out


# ---- ensemble members and gathered uploads ------------------------------------
def split_member_dim(op: Operand, ens_dim: str):
  """Removes `ens_dim` from the outer dims of `op`; returns (op', M, stride)."""
  if ens_dim not in op.outer_dims:
    raise ValueError(f'ensemble_dim={ens_dim!r} not found in {op.outer_dims}')
  i = op.outer_dims.index(ens_dim)
  m, stride = op.outer_shape[i], op.outer_strides[i]
  keep = [k for k in range(len(op.outer_dims)) if k != i]
  out = dataclasses.replace(
      op, outer_dims=tuple(op.outer_dims[k] for k in keep),
      outer_shape=tuple(op.outer_shape[k] for k in keep),
      outer_strides=tuple(op.outer_strides[k] for k in keep))
  terms = getattr(op, 'gather_terms', None)
  if terms is not None:
    # a gathered operand addresses through explicit (dims, offsets) terms: the
    # member axis must be a plain strided term
    rest = []
    for tdims, arr in terms:
      if ens_dim in tdims:
        if tdims != (ens_dim,):
          raise ValueError('the ensemble dimension cannot be part of a gather')
        arr = np.asarray(arr)
        stride = int(arr[1] - arr[0]) if arr.size > 1 else 0
        if arr.size > 2 and not (np.diff(arr) == stride).all():
          raise ValueError('ensemble members must be evenly strided')
      else:
        rest.append((tdims, arr))
    out.gather_terms = rest
  return out, int(m), int(stride)


def _upload_gathered(ctx: _lib.Context, op: Operand, staged: list) -> Operand:
  """Uploads ONLY the slabs a gathered host operand references (a by-init truth
  gather or a day-of-year climatology lookup addresses a few slabs of a long
  record: uploading the whole backing array, per variable and chunk, is what
  the round-1 review flagged), packed contiguously, and re-addresses the
  operand.  Dimensions that were plain strided terms (e.g. the ensemble
  members) stay plain strided terms of the packed copy, so that
  split_member_dim still sees an evenly strided member axis; the looked-up
  dimensions become one explicit offset term over the DISTINCT slabs."""
  terms = op.gather_terms
  plain, looked = [], []
  for tdims, arr in terms:
    arr = np.asarray(arr, dtype=np.int64)
    if len(tdims) == 1 and (arr.size < 2 or
                            (np.diff(arr) == arr[1] - arr[0]).all()):
      plain.append((tdims[0], arr))
    else:
      looked.append((tuple(tdims), arr))
  size = dict(zip(op.outer_dims, op.outer_shape))
  gdims = tuple(d for d in op.outer_dims if any(d in td for td, _ in looked))
  gshape = tuple(size[d] for d in gdims)
  goff = np.zeros(gshape, dtype=np.int64)
  for tdims, arr in looked:
    perm = [tdims.index(d) for d in gdims if d in tdims]
    a = np.transpose(arr, perm)
    a = a[tuple(slice(None) if d in tdims else None for d in gdims)]
    goff = goff + a
  uniq, inv = np.unique(goff.reshape(-1), return_inverse=True)
  slab = (op.nrow - 1) * op.row_stride + op.ncol
  pad = (slab + 63) // 64 * 64
  es = op.itemsize
  pshape = tuple(arr.size for _, arr in plain)
  nplain = int(np.prod(pshape)) if pshape else 1
  packed = np.empty((nplain, uniq.size, pad), dtype=op.dtype)
  grids = np.meshgrid(*[arr for _, arr in plain], indexing='ij') if plain else []
  poff = sum(grids).reshape(-1) if plain else np.zeros(1, np.int64)
  for pi in range(nplain):
    for ui, off in enumerate(uniq):
      src = np.ctypeslib.as_array(
          (np.ctypeslib.ctypes.c_char * (slab * es)).from_address(
              op.addr + (int(poff[pi]) + int(off)) * es)).view(op.dtype)
      packed[pi, ui, :slab] = src
  dptr = ctx.to_device(packed)
  staged.append(dptr)
  out = dataclasses.replace(op, addr=dptr, on_device=True)
  new_terms = []
  stride = uniq.size * pad
  for i in range(len(plain) - 1, -1, -1):
    d, arr = plain[i]
    new_terms.insert(0, ((d,), np.arange(arr.size, dtype=np.int64) * stride))
    stride *= arr.size
  if gdims:
    new_terms.append((gdims, (inv.astype(np.int64) * pad).reshape(gshape)))
  out.gather_terms = new_terms
  return out


# ---- launch plumbing -----------------------------------------------------------
class Staging:
  """Device copies of host operands for one launch, freed when the `with`
  block exits, also when the launch raises."""

  def __init__(self, ctx: _lib.Context):
    self.ctx = ctx
    self.ptrs: list = []

  def __enter__(self) -> 'Staging':
    return self

  def __exit__(self, *exc):
    for p in self.ptrs:
      self.ctx.free(p)

  def array(self, arr: np.ndarray) -> int:
    """Device copy of a host array."""
    ptr = self.ctx.to_device(arr)
    self.ptrs.append(ptr)
    return ptr

  def malloc(self, nbytes: int) -> int:
    """Uninitialised device buffer of `nbytes`."""
    ptr = self.ctx.malloc(nbytes)
    self.ptrs.append(ptr)
    return ptr

  def upload(self, op: Operand) -> Operand:
    """`op` re-addressed on the device: the smallest contiguous span of its
    backing array (same strides), or, for a gathered operand, only the slabs it
    references.  Device operands are returned as they are."""
    if op.on_device:
      return op
    if getattr(op, 'gather_terms', None) is not None:
      return _upload_gathered(self.ctx, op, self.ptrs)
    arr = op.data
    lo = arr.ctypes.data
    span = 1 + sum((n - 1) * abs(s) for n, s in zip(arr.shape, arr.strides)
                   ) // arr.itemsize if arr.size else 1
    flat = np.ctypeslib.as_array(
        (np.ctypeslib.ctypes.c_char * (span * arr.itemsize)).from_address(lo))
    out = dataclasses.replace(op, addr=self.array(flat), on_device=True)
    if hasattr(op, 'gather_terms'):
      out.gather_terms = op.gather_terms
    return out


_GRID = ('layout', 'nrow', 'ncol', 'row_stride')


def _check_grid(ops: Sequence[Operand], fields: tuple = _GRID, dtype=None):
  """Operands of one launch share one slab geometry: every operand agrees
  with the first on `fields` and, when given, has `dtype`."""
  first = ops[0]
  for op in ops[1:]:
    for f in fields:
      if getattr(op, f) != getattr(first, f):
        raise ValueError(f'operands of one launch must share {f}: '
                         f'{getattr(first, f)} vs {getattr(op, f)}')
  if dtype is not None:
    for op in ops:
      if op.dtype != dtype:
        raise ValueError(f'this kernel takes {np.dtype(dtype)} operands, not '
                         f'{op.dtype}')


def _check_truth(t_op: Operand, ens_dim: str):
  if ens_dim in t_op.outer_dims:
    raise ValueError(f'truth must not have the {ens_dim!r} dimension')


def addressing(ops: Sequence[Operand], dims: tuple, shape: tuple,
                base: Optional[int] = None):
  """(base, tables): the lowest address of `ops` (unless `base` is given) and
  the element offsets of every operand's slabs over the (dims, shape) grid,
  relative to it."""
  if base is None:
    base = min(op.addr for op in ops)
  tabs = []
  for op in ops:
    rel = op.addr - base
    assert rel % op.itemsize == 0
    tabs.append(offset_table(op, dims, shape) + rel // op.itemsize)
  return base, tabs


def _reduce_last(dims: tuple, shape: tuple, reduce_dim: Optional[str]):
  """The grid with `reduce_dim` (if present) moved last, for the map kernels
  that average over it: returns (dims, shape, out_dims, out_shape, ngroup)."""
  if reduce_dim is None or reduce_dim not in dims:
    return dims, shape, dims, shape, 1
  i = dims.index(reduce_dim)
  out_dims, out_shape = dims[:i] + dims[i + 1:], shape[:i] + shape[i + 1:]
  return (out_dims + (reduce_dim,), out_shape + (shape[i],), out_dims,
          out_shape, shape[i])


def _map_dims(op: Operand):
  return (LAT, LON) if op.layout == 'lat_lon' else (LON, LAT)


def run_region_groups(ctx: _lib.Context, groups, shape: tuple, axis: int,
                      launch, host: bool = False) -> np.ndarray:
  """Runs `launch(weights, out)` once per `build_weights` group and returns
  the float64 result of `shape`, whose axis `axis` indexes the regions.  Each
  launch writes the group's part (`shape` with that axis cut to the group)
  into a device buffer, or, with `host`, straight into host memory."""
  res = np.empty(shape, dtype=np.float64)
  for ids, spec in groups:
    part_shape = shape[:axis] + (len(ids),) + shape[axis + 1:]
    if host:
      part = np.empty(part_shape, dtype=np.float64)
      launch(spec, part.ctypes.data)
    else:
      out = ctx.malloc(int(np.prod(part_shape)) * 8)
      try:
        launch(spec, out)
        part = ctx.from_device(out, part_shape, np.float64)
      finally:
        ctx.free(out)
    res[(slice(None),) * axis + (ids,)] = part
  return res


def _run_maps(ctx: _lib.Context, forecast: Operand, truth: Operand,
              shape: tuple, dtype, launch):
  """Runs `launch(out)` into new output maps of `shape`.  They are a torch
  tensor left on the device when the forecast is a torch CUDA tensor (else
  when the truth is), otherwise NumPy copied back from a raw allocation."""
  src = forecast if xl._is_torch(forecast.data) else truth  # pylint: disable=protected-access
  if xl._is_torch(src.data):  # pylint: disable=protected-access
    import torch  # pylint: disable=import-outside-toplevel
    maps = torch.empty(shape, dtype=getattr(torch, np.dtype(dtype).name),
                       device=src.data.device)
    launch(int(maps.data_ptr()))
    return maps
  out = ctx.malloc(max(int(np.prod(shape)) * np.dtype(dtype).itemsize, 16))
  try:
    launch(out)
    return ctx.from_device(out, shape, dtype)
  finally:
    ctx.free(out)


# ---- K1: deterministic metrics -------------------------------------------------
def run_det_metrics(ctx: _lib.Context, f_ops: Sequence[Operand],
                    t_ops: Sequence[Operand],
                    c_ops: Optional[Sequence[Operand]], latitude, longitude,
                    regions: Sequence, skipna: bool, cell_cache=None):
  """Runs K1 for a list of variables that share dtype / layout / grid.

  Returns (stats, dims, shapes): stats[v] has shape outer_shape[v] +
  (len(regions), DET_NSTAT).
  """
  first = f_ops[0]
  all_ops = list(f_ops) + list(t_ops) + (list(c_ops) if c_ops else [])
  _check_grid(all_ops, _GRID + ('on_device', 'dtype'))
  base = min(op.addr for op in all_ops)
  dims_list, shape_list, tabs = [], [], [[], [], []]
  for v in range(len(f_ops)):
    trio = [f_ops[v], t_ops[v]] + ([c_ops[v]] if c_ops else [])
    dims, shape = broadcast_dims(*trio)
    dims_list.append(dims)
    shape_list.append(shape)
    for k, tab in enumerate(addressing(trio, dims, shape, base)[1]):
      tabs[k].append(tab)
  off_f, off_t, off_c = (np.ascontiguousarray(np.concatenate(t)) if t else None
                         for t in tabs)
  c = base if c_ops else None
  code = _lib.F32 if first.dtype == np.float32 else _lib.F64
  nreg = len(regions)
  groups = build_weights(ctx, np.asarray(latitude), np.asarray(longitude),
                         regions, first.layout, first.row_stride, cell_cache)
  host = not first.on_device
  result = run_region_groups(
      ctx, groups, (off_f.size, nreg, _lib.DET_NSTAT), 1,
      lambda w, out: ctx.det_metrics(base, base, c, code, off_f, off_t, off_c,
                                     w, skipna, out, host=host), host)
  stats, pos = [], 0
  for shape in shape_list:
    n = int(np.prod(shape)) if shape else 1
    stats.append(result[pos:pos + n].reshape(shape + (nreg, _lib.DET_NSTAT)))
    pos += n
  return stats, dims_list, shape_list


# ---- K2: ensemble metrics ----------------------------------------------------
def run_ens_metrics(ctx: _lib.Context, x_ops: Sequence[Operand],
                    t_ops: Sequence[Operand], ens_dim: str, latitude,
                    longitude, regions: Sequence, skipna: bool,
                    cell_cache=None):
  """Runs K2 for variables sharing layout / grid.  Returns (stats, dims,
  shapes, M): stats[v] has shape outer_shape[v] + (len(regions), ENS_NSTAT)."""
  # all-host float32 operands: stream member / truth slabs through the staging
  # buffers (wb2_ens_metrics_host; truth slabs go through the slab cache)
  host = all(not o.on_device and o.dtype == np.float32
             for o in list(x_ops) + list(t_ops))
  with Staging(ctx) as stage:
    pairs = []
    for xo, to in zip(x_ops, t_ops):
      _check_truth(to, ens_dim)
      if not host:
        xo, to = stage.upload(xo), stage.upload(to)
      pairs.append(split_member_dim(xo, ens_dim) + (to,))
    first = pairs[0][0]
    nreg = len(regions)
    groups = build_weights(ctx, np.asarray(latitude), np.asarray(longitude),
                           regions, first.layout, first.row_stride, cell_cache)
    stats, dims_list, shape_list, ms = [], [], [], []
    for xo, m, st, to in pairs:
      _check_grid([xo, to])
      # xarray puts truth's dims first for abs(truth - forecast)
      # (metrics.py:824); we keep the forecast-first order used by every other
      # metric of this module and of the reference's `mean/var` based ones.
      dims, shape = broadcast_dims(xo, to)
      base, (off_x, off_t) = addressing([xo, to], dims, shape)
      if host:
        launch = lambda w, out: ctx.ens_metrics_host(  # pylint: disable=cell-var-from-loop
            base, base, m, st, off_x, off_t, w, skipna, out)
      else:
        launch = lambda w, out: ctx.ens_metrics(  # pylint: disable=cell-var-from-loop
            base, base, _lib.F32, m, st, off_x, off_t, w, skipna, out)
      res = run_region_groups(ctx, groups, (off_x.size, nreg, _lib.ENS_NSTAT),
                              1, launch, host)
      stats.append(res.reshape(shape + (nreg, _lib.ENS_NSTAT)))
      dims_list.append(dims)
      shape_list.append(shape)
      ms.append(m)
  return stats, dims_list, shape_list, ms


# ---- K3: energy score --------------------------------------------------------
ENERGY_MAX_REGIONS = _lib.MAX_REGIONS


def run_energy_score(ctx: _lib.Context, x_ops: Sequence[Operand],
                     t_ops: Sequence[Operand], ens_dim: str, latitude,
                     longitude, regions: Sequence, cell_cache=None):
  """Runs K3.  Returns (stats, dims, M): stats[v] has shape
  outer_shape[v] + (len(regions), 4, M) -- see wb2_energy_score."""
  groups = None
  stats, dims_list, ms = [], [], []
  with Staging(ctx) as stage:
    for xo, to in zip(x_ops, t_ops):
      xo, to = stage.upload(xo), stage.upload(to)
      xo, m, st = split_member_dim(xo, ens_dim)
      if groups is None:
        groups = build_weights(ctx, np.asarray(latitude),
                               np.asarray(longitude), regions, xo.layout,
                               xo.row_stride, cell_cache, ENERGY_MAX_REGIONS)
      dims, shape = broadcast_dims(xo, to)
      base, (off_x, off_t) = addressing([xo, to], dims, shape)
      res = run_region_groups(
          ctx, groups, (off_x.size, len(regions), 4, m), 1,
          lambda w, out: ctx.energy_score(  # pylint: disable=cell-var-from-loop
              base, base, _lib.F32, m, st, off_x, off_t, w, out))
      stats.append(res.reshape(shape + (len(regions), 4, m)))
      dims_list.append(dims)
      ms.append(m)
  return stats, dims_list, ms


# ---- K6: map-output metrics (time mean fused in) -------------------------------
def run_det_maps(ctx: _lib.Context, f_op: Operand, t_op: Operand, stat: int,
                 reduce_dim: Optional[str], skipna: bool):
  """Runs K6 for one variable: maps of stat(f, t) averaged over `reduce_dim`
  (None: no averaging).  Returns (maps, dims)."""
  with Staging(ctx) as stage:
    f_op, t_op = stage.upload(f_op), stage.upload(t_op)
    _check_grid([f_op, t_op], _GRID + ('dtype',))
    dims, shape, out_dims, out_shape, ngroup = _reduce_last(
        *broadcast_dims(f_op, t_op), reduce_dim)
    base, (off_f, off_t) = addressing([f_op, t_op], dims, shape)
    code = _lib.F32 if f_op.dtype == np.float32 else _lib.F64
    maps = _run_maps(
        ctx, f_op, t_op, out_shape + (f_op.nrow, f_op.ncol), f_op.dtype,
        lambda out: ctx.det_maps(base, base, code, stat, off_f.size // ngroup,
                                 ngroup, off_f, off_t, f_op.nrow, f_op.ncol,
                                 f_op.row_stride, skipna, out))
  return maps, out_dims + _map_dims(f_op)


def run_ens_maps(ctx: _lib.Context, x_op: Operand, t_op: Operand,
                 ens_dim: str, stat_mask: int, reduce_dim: Optional[str],
                 skipna: bool):
  """Runs K6e for one variable.  Returns (maps[nsel, ...], dims, M): the
  selected point-wise ensemble statistics (increasing bit order of
  `stat_mask`) averaged over `reduce_dim`."""
  _check_truth(t_op, ens_dim)
  with Staging(ctx) as stage:
    x_op, t_op = stage.upload(x_op), stage.upload(t_op)
    x_op, m, st = split_member_dim(x_op, ens_dim)
    _check_grid([x_op, t_op], dtype=np.float32)
    dims, shape, out_dims, out_shape, ngroup = _reduce_last(
        *broadcast_dims(x_op, t_op), reduce_dim)
    base, (off_x, off_t) = addressing([x_op, t_op], dims, shape)
    nsel = bin(stat_mask).count('1')
    maps = _run_maps(
        ctx, x_op, t_op, (nsel,) + out_shape + (x_op.nrow, x_op.ncol),
        np.float32,
        lambda out: ctx.ens_maps(base, base, _lib.F32, m, st,
                                 off_x.size // ngroup, ngroup, off_x, off_t,
                                 x_op.nrow, x_op.ncol, x_op.row_stride,
                                 stat_mask, skipna, out))
  return maps, out_dims + _map_dims(x_op), m


# ---- K7: threshold / Gaussian metrics -----------------------------------------
THR_NOUT = 8


def _threshold_operands(spec, stage: Staging):
  """Stages the threshold operands of `spec`: ('field', [op per threshold]),
  ('gaussian', mean_op, std_op, [z]) or None (no thresholds).  Returns (ops,
  args): args(base, tables) -> the kernel's (nq, thr_a, off_a, thr_b, off_b,
  z) from the offset tables of `ops` relative to `base`."""
  if spec is None:
    return [], lambda base, tabs: (0, None, None, None, None, None)
  if spec[0] == 'gaussian':
    ops = [stage.upload(spec[1]), stage.upload(spec[2])]
    z = np.asarray(spec[3], dtype=np.float64)
    return ops, lambda base, tabs: (z.size, base, tabs[0], base, tabs[1], z)
  seen: dict = {}  # thresholds that share a climatology array share its upload

  def one(op):
    if op.on_device or getattr(op, 'gather_terms', None) is not None:
      # a gathered threshold field (day-of-year / quantile lookup): only the
      # slabs it references are uploaded, re-addressed by the returned operand
      return stage.upload(op)
    key = id(op.data)
    if key not in seen:
      seen[key] = stage.upload(op).addr
    return dataclasses.replace(op, addr=seen[key], on_device=True)

  ops = [one(op) for op in spec[1]]
  return ops, lambda base, tabs: (
      len(ops), base, np.ascontiguousarray(np.concatenate(tabs)), None, None,
      None)


def run_ens_threshold_metrics(ctx: _lib.Context, x_op: Operand, t_op: Operand,
                              ens_dim: str, spec, latitude, longitude,
                              regions: Sequence, skipna: bool,
                              cell_cache=None):
  """Runs K7 (ensemble entry) for one variable.  Returns (stats, dims, M):
  stats has shape outer_shape + (nq, len(regions), 8)."""
  _check_truth(t_op, ens_dim)
  with Staging(ctx) as stage:
    x_op, t_op = stage.upload(x_op), stage.upload(t_op)
    x_op, m, st = split_member_dim(x_op, ens_dim)
    dims, shape = broadcast_dims(x_op, t_op)
    thr_ops, thr_args = _threshold_operands(spec, stage)
    _check_grid([x_op, t_op] + thr_ops, dtype=np.float32)
    base, tabs = addressing([x_op, t_op] + thr_ops, dims, shape)
    nq, *thr = thr_args(base, tabs[2:])
    nreg = len(regions)
    groups = build_weights(ctx, np.asarray(latitude), np.asarray(longitude),
                           regions, x_op.layout, x_op.row_stride, cell_cache)
    res = run_region_groups(
        ctx, groups, (tabs[0].size, nq, nreg, THR_NOUT), 2,
        lambda w, out: ctx.ens_threshold_metrics(
            base, base, m, st, tabs[0], tabs[1], nq, *thr, w, skipna, out))
  return res.reshape(shape + (nq, nreg, THR_NOUT)), dims, m


def run_gaussian_metrics(ctx: _lib.Context, m_op: Operand, s_op: Operand,
                         t_op: Operand, spec, latitude, longitude,
                         regions: Sequence, skipna: bool, cell_cache=None):
  """Runs K7 (Gaussian entry) for one variable; spec None -> CRPS / variance.
  Returns (stats, dims): stats has shape outer_shape + (max(nq, 1), R, 8)."""
  with Staging(ctx) as stage:
    ops = [stage.upload(op) for op in (m_op, s_op, t_op)]
    dims, shape = broadcast_dims(*ops)
    thr_ops, thr_args = _threshold_operands(spec, stage)
    _check_grid(ops + thr_ops, dtype=np.float32)
    base, tabs = addressing(ops + thr_ops, dims, shape)
    nq, *thr = thr_args(base, tabs[3:])
    nq_out = max(nq, 1)
    nreg = len(regions)
    groups = build_weights(ctx, np.asarray(latitude), np.asarray(longitude),
                           regions, ops[0].layout, ops[0].row_stride,
                           cell_cache)
    res = run_region_groups(
        ctx, groups, (tabs[0].size, nq_out, nreg, THR_NOUT), 2,
        lambda w, out: ctx.gaussian_metrics(base, base, base, *tabs[:3], nq,
                                            *thr, w, skipna, out))
  return res.reshape(shape + (nq_out, nreg, THR_NOUT)), dims


def run_ens_threshold_maps(ctx: _lib.Context, x_op: Operand, t_op: Operand,
                           ens_dim: str, spec, stat: int,
                           reduce_dim: Optional[str], skipna: bool):
  """Runs the map-output form of K7 for one variable.  Returns (maps, dims,
  M): maps[nq, ...outer (without reduce_dim)..., nrow, ncol] float32."""
  _check_truth(t_op, ens_dim)
  with Staging(ctx) as stage:
    x_op, t_op = stage.upload(x_op), stage.upload(t_op)
    x_op, m, st = split_member_dim(x_op, ens_dim)
    dims, shape, out_dims, out_shape, ngroup = _reduce_last(
        *broadcast_dims(x_op, t_op), reduce_dim)
    thr_ops, thr_args = _threshold_operands(spec, stage)
    _check_grid([x_op, t_op] + thr_ops, dtype=np.float32)
    base, tabs = addressing([x_op, t_op] + thr_ops, dims, shape)
    nq, *thr = thr_args(base, tabs[2:])
    maps = _run_maps(
        ctx, x_op, t_op, (nq,) + out_shape + (x_op.nrow, x_op.ncol),
        np.float32,
        lambda out: ctx.ens_threshold_maps(
            base, base, m, st, tabs[0].size // ngroup, ngroup, tabs[0],
            tabs[1], nq, *thr, x_op.nrow, x_op.ncol, x_op.row_stride, stat,
            skipna, out))
  return maps, out_dims + _map_dims(x_op), m


# ---- K9: SEEPS maps, K10: rank histogram ------------------------------------------
def run_seeps_maps(ctx: _lib.Context, f_op: Operand, t_op: Operand,
                   wet_op: Operand, f_lookup: dict, t_lookup: dict, p1,
                   dry_threshold: float, min_p1: float, max_p1: float,
                   reduce_dim: Optional[str], skipna: bool):
  """Runs K9 for one variable: SEEPS maps of (f, t) averaged over
  `reduce_dim`.  The wet thresholds `wet_op` are looked up at the forecast's
  and the truth's valid times through the `gather_operand` index maps
  `f_lookup` / `t_lookup`; `p1` is the (latitude, longitude) DataArray of the
  average dry fraction.  Every operand keeps its dtype (float32 or float64):
  the kernel compares in NumPy's promoted dtype, as the reference does.
  Returns (maps, dims)."""
  p1 = np.asarray(p1.transpose(*_map_dims(f_op)).values)
  for what, dt in (('forecast', f_op.dtype), ('truth', t_op.dtype),
                   ('wet threshold', wet_op.dtype), ('dry fraction', p1.dtype)):
    if dt not in (np.float32, np.float64):
      raise TypeError(f'SEEPS takes float32 or float64 data; the {what} is '
                      f'{dt}')
  p1 = np.ascontiguousarray(p1)
  if p1.shape != (f_op.nrow, f_op.ncol):
    raise ValueError(f'dry fraction grid {p1.shape} does not match the '
                     f'data grid {(f_op.nrow, f_op.ncol)}')
  # The Python-float thresholds are weak scalars: rounded to the dtype they
  # are compared in, the dry threshold to the precipitation's (the kernel
  # rounds it again for a float32 side of a mixed pair, which changes
  # nothing) and the p1 bounds to p1's.  Only float64 operands are named, so
  # an all-float32 launch makes the same Context call, with the same values,
  # as before the dtype codes existed.
  dry_threshold = float(np.result_type(f_op.dtype, t_op.dtype).type(
      dry_threshold))
  min_p1, max_p1 = (float(p1.dtype.type(v)) for v in (min_p1, max_p1))
  dtypes = {f'{k}_dtype': _lib.F64 for k, dt in (
      ('f', f_op.dtype), ('t', t_op.dtype), ('wet', wet_op.dtype),
      ('p1', p1.dtype)) if dt == np.float64}
  with Staging(ctx) as stage:
    f_op, t_op, wet_op = (stage.upload(op) for op in (f_op, t_op, wet_op))
    _check_grid([f_op, t_op])
    # the threshold climatology keeps its own row stride
    _check_grid([f_op, wet_op], ('nrow', 'ncol'))
    ops = [f_op, t_op, gather_operand(wet_op, f_lookup),
           gather_operand(wet_op, t_lookup)]
    dims, shape, out_dims, out_shape, ngroup = _reduce_last(
        *broadcast_dims(*ops), reduce_dim)
    tabs = [offset_table(op, dims, shape) for op in ops]
    p1_dev = stage.array(p1)
    maps = _run_maps(
        ctx, f_op, t_op, out_shape + (f_op.nrow, f_op.ncol), np.float32,
        lambda out: ctx.seeps_maps(
            f_op.addr, t_op.addr, wet_op.addr, p1_dev, tabs[0].size // ngroup,
            ngroup, *tabs, f_op.nrow, f_op.ncol, f_op.row_stride,
            wet_op.row_stride, float(dry_threshold), float(min_p1),
            float(max_p1), skipna, out, **dtypes))
  return maps, out_dims + _map_dims(f_op)


def run_rank_histogram(ctx: _lib.Context, x_op: Operand, t_op: Operand,
                       ens_dim: str, nbins: int, reduce_dim: Optional[str],
                       random_ties: bool, seed: int):
  """Runs K10 for one variable.  Returns (hist[..., nrow, ncol, nbins], dims
  without `bins`)."""
  _check_truth(t_op, ens_dim)
  with Staging(ctx) as stage:
    x_op, t_op = stage.upload(x_op), stage.upload(t_op)
    x_op, nmember, stride = split_member_dim(x_op, ens_dim)
    _check_grid([x_op, t_op])
    dims, shape, out_dims, out_shape, ngroup = _reduce_last(
        *broadcast_dims(x_op, t_op), reduce_dim)
    off_x, off_t = (offset_table(op, dims, shape) for op in (x_op, t_op))
    hist = _run_maps(
        ctx, x_op, t_op, out_shape + (x_op.nrow, x_op.ncol, nbins), np.float32,
        lambda out: ctx.rank_histogram(
            x_op.addr, t_op.addr, nmember, stride, off_x.size // ngroup,
            ngroup, off_x, off_t, x_op.nrow, x_op.ncol, x_op.row_stride, nbins,
            random_ties, seed, out))
  return hist, out_dims + _map_dims(x_op)

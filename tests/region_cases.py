"""Seeded raw-ABI cases for the region-weighted reduction every metric kernel
shares (csrc/region_reduce.cuh): K1 LDG / TMA / TMA-seg, K2 pair / twin /
scalar, K2b (ens_big), K3 (energy) and the *_host entries.

Exact family.  Inputs are multiples of 2^-1 in [-1, 1] and every weight
factor (row_w, seg_w, col_w, cell_w) is 0 or +-2^-j for small j, so every
product in the reduction is exact, the TMA-seg path's float32 row_c =
max_r |row_w| and pattern = row_w / row_c are powers of two, and every sum is
exact as long as its terms span at most 24 (float32 accumulators) or 53
(float64) bits.  `bit_budget` computes that span per accumulator and path; the
CPU test asserts it, which is what makes bit equality with the float64
reference the right assertion on the GPU.  Exact slots: every K1 and K3 slot;
K2 / K2b skill, mse and the weight sums when M is a power of two (spread,
variance and debiased MSE carry a rounding by 1 / (M - 1): `ens_bound`).

Every element no slab reads is a NaN sentinel: row padding, gaps between
slabs and members, one element before the first slab and after the last.  An
out-of-range read turns an exact result into NaN.

`plan` mirrors the host dispatch (det_metrics.cu det_metrics_impl, det_tma.cu
det_metrics_tma / det_metrics_tma_seg, ens_metrics.cu try_pair / launch_ens,
ens_energy.cu, host_stream.cu) and predicts the path and the launch count.
The launch count is observable through wb2_launch_count; which kernel ran is
not (TMA and LDG both make two launches), so for that choice this model is
the evidence, and it is kept line for line with the host code."""
from __future__ import annotations

import dataclasses
from typing import Optional

import numpy as np

NUM_SMS = 132  # H100 SXM; the grid-regime claims below assume it
U = 2.0 ** -24
DET_NSTAT = 10
ENS_NSTAT = 10
PAIR_MP = (2, 3, 4, 5, 8, 10, 16, 20, 32, 50, 64)  # launch_ens buckets


@dataclasses.dataclass
class Case:
  name: str
  kind: str                  # det | vector | ens | energy
  nrow: int
  ncol: int
  row_stride: int
  row_w: np.ndarray          # [R][nrow] float64
  seg_start: np.ndarray      # [nseg + 1] int32
  seg_w: np.ndarray          # [R][nseg] float64
  col_w: Optional[np.ndarray] = None   # [ncol] float32
  cell_w: Optional[np.ndarray] = None  # [nrow][ncol] float32 (uploaded)
  zero_skip: bool = True
  skipna: bool = False
  dtype: type = np.float32
  clim: bool = False
  nmember: int = 0
  member_stride: int = 0
  buffers: dict = dataclasses.field(default_factory=dict)  # name -> 1-D array
  offsets: dict = dataclasses.field(default_factory=dict)  # name -> int64[nfield]
  slabs: dict = dataclasses.field(default_factory=dict)    # name -> slab starts
  env: tuple = ({},)          # forced-path variants the GPU test runs
  host: bool = False          # through wb2_*_host
  stage_mb: int = 0           # WB2_STAGE_MB on a fresh context (host only)
  covers: tuple = ()
  exact: bool = True
  cell_w_dev: Optional[int] = None    # realistic family: build_weights' upload

  @property
  def nregion(self):
    return self.row_w.shape[0]

  @property
  def nseg(self):
    return self.seg_start.size - 1

  @property
  def nfield(self):
    return next(iter(self.offsets.values())).size

  def weight_spec(self, cell_w_dev=None):
    from weatherbench2_b200 import _lib  # pylint: disable=import-outside-toplevel
    return _lib.WeightSpec(self.nrow, self.ncol, self.row_w, self.seg_start,
                           self.seg_w, self.col_w, cell_w_dev, self.zero_skip,
                           self.row_stride)

  def dense_w(self):
    """W[r, row, col] of include/wb2b200.h (wb2_weights), in float64."""
    seg = np.repeat(np.arange(self.nseg), np.diff(self.seg_start))
    w = self.row_w[:, :, None] * self.seg_w[:, seg][:, None, :]
    if self.col_w is not None:
      w = w * self.col_w.astype(np.float64)[None, None, :]
    if self.cell_w is not None:
      w = w * self.cell_w.astype(np.float64)[None]
    return w

  def slab(self, name, start):
    b = self.buffers[name]
    idx = (start + np.arange(self.nrow)[:, None] * self.row_stride +
           np.arange(self.ncol)[None, :])
    return b[idx].astype(np.float64)

  def fields(self, name):
    """[nfield, nrow, ncol] float64 slabs of operand `name` (members of an
    ensemble: [nfield, M, nrow, ncol])."""
    off = self.offsets[name]
    if name == 'x':
      return np.stack([np.stack([self.slab('x', o + m * self.member_stride)
                                 for m in range(self.nmember)]) for o in off])
    return np.stack([self.slab(name, o) for o in off])


# ---- building blocks -----------------------------------------------------------
def _grid(rs, shape, step=0.5, lim=1.0):
  n = int(round(lim / step))
  return rs.randint(-n, n + 1, size=shape).astype(np.float64) * step


def _pow2(rs, shape, jmax=3, pzero=0.0, neg=False):
  shape = tuple(np.atleast_1d(shape))
  w = 2.0 ** -rs.randint(0, jmax + 1, size=shape)
  if pzero:
    w = np.where(rs.rand(*shape) < pzero, 0.0, w)
  if neg:
    w = w * np.where(rs.rand(*shape) < 0.4, -1.0, 1.0)
  return w


def _place(nslab, span, align=4, shift=0, gap=3):
  """Starts of `nslab` slabs of `span` elements, each start a multiple of
  `align` plus `shift`, with at least `gap` sentinel elements between them and
  at least one before the first and after the last; returns (starts, length)."""
  starts, pos = [], 1
  for _ in range(nslab):
    s = (pos + align - 1 - shift) // align * align + shift
    while s < pos:
      s += align
    starts.append(s)
    pos = s + span + gap
  return np.array(starts, np.int64), pos + 1


def _fill(dtype, length, starts, nrow, ncol, row_stride, values):
  """NaN buffer with values[i] ([nrow, ncol]) written at slab i."""
  buf = np.full(length, np.nan, dtype=dtype)
  for s, v in zip(starts, values):
    idx = s + np.arange(nrow)[:, None] * row_stride + np.arange(ncol)[None, :]
    buf[idx] = v
  return buf


def _weights(rs, nrow, ncol, nregion, seg_start, *, jmax=3, row_zero=0.25,
             seg_zero=0.25, neg=False, first_full=True, dead=True):
  """Random dyadic row_w / seg_w.  first_full: region 0 weighs every cell
  but the `dead` ones; dead: one row (nrow >= 3) and one segment (nseg >= 2)
  that no region weighs, so the zero_skip branches of every kernel run."""
  nseg = len(seg_start) - 1
  row_w = _pow2(rs, (nregion, nrow), jmax, row_zero, neg)
  seg_w = _pow2(rs, (nregion, nseg), jmax, seg_zero, neg)
  if first_full:
    row_w[0] = np.abs(row_w[0]) + (row_w[0] == 0)
    seg_w[0] = np.abs(seg_w[0]) + (seg_w[0] == 0)
  if dead and nrow >= 3:
    row_w[:, rs.randint(nrow)] = 0.0
  if dead and nseg >= 2:
    seg_w[:, rs.randint(nseg)] = 0.0
  return row_w, np.asarray(seg_start, np.int32), seg_w


def _banded_row_w(rs, nrow, nregion, nband, jmax=3):
  """row_w whose normalised region pattern changes exactly nband - 1 times:
  row_c varies inside a band, the pattern does not."""
  cuts = np.sort(rs.choice(np.arange(1, nrow), nband - 1, replace=False))
  bands = np.split(np.arange(nrow), cuts)
  w = np.zeros((nregion, nrow))
  prev = None
  for rows in bands:
    while True:
      pat = _pow2(rs, nregion, jmax, 0.3)
      pat[rs.randint(nregion)] = 1.0
      if prev is None or not np.array_equal(pat, prev):
        break
    prev = pat
    for row in rows:
      w[:, row] = pat * 2.0 ** -rs.randint(0, 3)
  return w


def _poison(case, rs, values):
  """Without skipna, NaN and Inf must propagate into exactly the regions
  that weigh their cell.  Field 0: NaN in up to two cells that some regions
  weigh and others do not (every region if there is no such cell); field 1:
  +Inf in one such cell (K1 only: an Inf member makes K2's mean-removed sort
  NaN where the reference has Inf); the last of >= 3 fields: NaN in a cell
  every region weighs."""
  W = case.dense_w()
  some = (W != 0).any(axis=0) & (W == 0).any(axis=0)
  every = (W != 0).all(axis=0)
  name = 'x' if 'x' in values else 'f'
  v = values[name]
  nf = v.shape[0]

  def put(field, pool, k, val):
    cells = np.argwhere(pool)
    if not cells.size:
      return
    for r, c in cells[rs.choice(len(cells), min(k, len(cells)), replace=False)]:
      if v.ndim == 4:
        v[field, rs.randint(v.shape[1]), r, c] = val
      else:
        v[field, r, c] = val

  put(0, some if some.any() else every, 2, np.nan)
  if nf > 1 and name == 'f':
    put(1, some, 1, np.inf)
  if nf > 2:
    put(nf - 1, every, 1, np.nan)


def _finish(case, rs, values, nan_cells=None, sentinel_in_zero=True,
            poison=True):
  """Lays out the operands of `case` (values: name -> [nfield, (M,) nrow, ncol])
  and stores buffers / offsets.  nan_cells: operand name -> [nfield, nrow,
  ncol] bool of the cells that hold NaN in that operand (skipna cases);
  poison: see _poison (cases without skipna)."""
  values = {k: v.copy() for k, v in values.items()}
  if poison and not case.skipna:
    _poison(case, rs, values)
  W = case.dense_w()
  allzero = (W == 0).all(axis=0) if case.zero_skip else np.zeros(W.shape[1:], bool)
  span = (case.nrow - 1) * case.row_stride + case.ncol
  align = case.__dict__.pop('_align', 4)
  shift = case.__dict__.pop('_shift', 0)
  for k, (name, v) in enumerate(values.items()):
    v = v.copy()
    if nan_cells is not None and name in nan_cells:
      v = np.where(nan_cells[name], np.nan, v)
    if sentinel_in_zero and allzero.any():
      # cells no region weighs hold NaN / Inf: zero_skip must drop them
      bad = np.where(rs.rand(*allzero.shape) < 0.5, np.nan, np.inf)
      v = np.where(allzero, bad, v)
    if name == 'x':
      M = case.nmember
      ms = case.member_stride
      starts, length = _place(v.shape[0], (M - 1) * ms + span, align, shift)
      buf = np.full(length, np.nan, dtype=case.dtype)
      slabs = []
      for i, s in enumerate(starts):
        for m in range(M):
          slabs.append(s + m * ms)
      buf = _fill(case.dtype, length, slabs, case.nrow, case.ncol,
                  case.row_stride, v.reshape(-1, case.nrow, case.ncol))
      case.slabs[name] = np.array(slabs, np.int64)
    else:
      starts, length = _place(v.shape[0], span, align, shift)
      buf = _fill(case.dtype, length, starts, case.nrow, case.ncol,
                  case.row_stride, v)
      case.slabs[name] = starts
    case.buffers[name] = buf
    case.offsets[name] = starts
  return case


# ---- dispatch model ----------------------------------------------------------------
@dataclasses.dataclass
class Plan:
  path: str            # ldg | tma | tma_seg | pair | twin | scalar | big | energy
  launches: int
  vec: int = 1
  chunks: int = 0
  bands: tuple = ()
  rounds: tuple = ()   # lane rounds per half row (TMA-seg)
  cw: int = 0
  rows_per_block: int = 0
  gs: int = 0
  vec4: bool = False
  groups: int = 1


def block_rows(nrow, nfield, rows, min_rows, min_ctas):
  nblk = -(-nrow // rows)
  while nblk * nfield < min_ctas and rows > min_rows:
    rows = max(min_rows, rows // 2)
    nblk = -(-nrow // rows)
  return rows, nblk


def _offsets_multiple(case, m, names):
  return all((case.offsets[n] % m == 0).all() for n in names)


def seg_spans(ncol, seg_start):
  """det_metrics_tma_seg's spans: (nspan per half) or None (LDG fallback)."""
  half_cols = (ncol + 1) // 2
  out = []
  for half in (0, 1):
    h0, h1 = (half_cols, ncol) if half else (0, half_cols)
    best = []
    for limit in (32, 64):
      for S in range(max(1, -(-(h1 - h0) // limit)), h1 - h0 + 1):
        cur = 0
        for k in range(len(seg_start) - 1):
          a, b = max(h0, seg_start[k]), min(h1, seg_start[k + 1])
          if a < b:
            cur += -(-(b - a) // S)
        if cur <= limit:
          best = [cur]
          break
      if best:
        break
    if not best and h1 > h0:
      return None
    out.append(best[0] if best else 0)
  return out


def seg_bands(row_w, rch):
  """Bands per region chunk, or None when a chunk has more than 128."""
  R, nrow = row_w.shape
  out = []
  for r0 in range(0, R, rch):
    w = row_w[r0:r0 + rch]
    cmax = np.abs(w).max(axis=0)
    pat = np.where(cmax > 0, w / np.where(cmax > 0, cmax, 1), 0).astype(np.float32)
    n = 1 + int((pat[:, 1:] != pat[:, :-1]).any(axis=0).sum())
    if n > 128:
      return None
    out.append(n)
  return out


def _det_plan(case, env, offsets_aligned=None):
  nf = case.nfield
  f32 = case.dtype == np.float32
  vec = 4 if f32 else 2
  names = ['f', 't'] + (['c'] if case.clim else []) + (
      ['fv', 'tv'] if case.kind == 'vector' else [])
  aligned = (_offsets_multiple(case, vec, names) if offsets_aligned is None
             else offsets_aligned)
  vec_ok = case.row_stride % vec == 0 and aligned
  weighted = case.col_w is not None or case.cell_w is not None
  rows, _ = block_rows(case.nrow, nf, 32, 8, 2 * NUM_SMS)
  ldg = Plan('ldg', 2, vec if vec_ok else 1, rows_per_block=rows)
  if (env.get('WB2_DET_PATH') == 'ldg' or not f32 or not vec_ok or weighted or
      case.ncol % 4 or case.kind == 'vector'):
    return ldg
  noper = 3 if case.clim else 2
  if case.ncol * 4 < 512:
    return ldg
  stage_op = (case.ncol * 4 + 127) // 128 * 128
  if case.nseg == 1:
    nstage = min(32, (220 * 1024 // (noper * stage_op)) // 4 * 4)
    return Plan('tma', 2) if nstage >= 8 else ldg
  cw = 8
  rch = 8 if case.skipna else 16
  ns = (6 if case.clim else 3) + ((4 if case.clim else 1) if case.skipna else 1)
  bands = seg_bands(case.row_w, rch)
  if bands is None:
    return ldg
  fixed = (cw * rch * ns * 8 + case.nseg * rch * 4 + (case.nseg + 1) * 4 +
           128 * rch * 4 + 256)
  if fixed >= 220 * 1024:
    return ldg
  nstage = min(32, (220 * 1024 - fixed) // (noper * stage_op + 16))
  if nstage < cw // 2 + 3:
    return ldg
  spans = seg_spans(case.ncol, case.seg_start)
  if spans is None:
    return ldg
  k = len(bands)
  return Plan('tma_seg', 2 if k == 1 else 3 * k, chunks=k, bands=tuple(bands),
              rounds=tuple(1 if s <= 32 else 2 for s in spans), cw=cw)


def _ens_plan(case, env):
  M = case.nmember
  if M > 64:
    return Plan('big', 2)
  mp = next(b for b in PAIR_MP if M <= b)
  exact = M == mp
  weighted = case.col_w is not None or case.cell_w is not None
  aligned8 = _offsets_multiple(case, 2, ['x', 't'])
  rows, _ = block_rows(case.nrow, case.nfield, 8, 4, 4 * NUM_SMS)
  if (mp >= 8 and mp % 2 == 0 and env.get('WB2_ENS_PATH') != 'scalar' and
      not case.skipna and exact and aligned8 and case.nseg == 1 and
      not weighted and case.ncol % 2 == 0 and case.row_stride % 2 == 0 and
      case.member_stride % 2 == 0):
    return Plan('pair', 2, rows_per_block=rows)
  if (exact and not case.skipna and mp >= 8 and mp % 2 == 0 and
      env.get('WB2_ENS_SORT') != 'exact'):
    return Plan('twin', 2, rows_per_block=rows)
  return Plan('scalar', 2, rows_per_block=rows)


def _energy_plan(case):
  M = case.nmember
  gs = 4 if M <= 4 else 8
  ng = -(-M // gs)
  rif = max(1, 8 // ng)
  rows, _ = block_rows(case.nrow, case.nfield, 8 * rif, rif, 4 * NUM_SMS)
  vec4 = (case.member_stride % 4 == 0 and case.row_stride % 4 == 0 and
          all(s % 4 == 0 for s in case.seg_start) and
          _offsets_multiple(case, 4, ['x', 't']))
  weighted = case.col_w is not None or case.cell_w is not None
  return Plan('energy', 2, gs=gs, vec4=vec4 and not weighted,
              rows_per_block=rows)


def host_groups(case):
  """Staging groups of wb2_det_metrics_host / wb2_ens_metrics_host (no slab
  cache, distinct slab addresses)."""
  es = np.dtype(case.dtype).itemsize
  span = (case.nrow - 1) * case.row_stride + case.ncol
  slab_bytes = -(-span // 64) * 64 * es
  cap = (case.stage_mb or 256) << 20
  if case.kind == 'ens':
    per = case.nmember + 1
    cap = max(cap, slab_bytes * per)
    fpg = max(1, (cap // slab_bytes) // per)
  else:
    noper = 3 if case.clim else 2
    cap = max(cap, slab_bytes * 2 * noper)
    fpg = (cap // slab_bytes - noper) // noper
  return -(-case.nfield // fpg)


def plan(case, env=None):
  env = env or {}
  if case.kind in ('det', 'vector'):
    if case.host:  # staged slabs start at multiples of 64 elements
      p = _det_plan(case, env, offsets_aligned=True)
      g = host_groups(case)
      return dataclasses.replace(p, launches=p.launches * g, groups=g)
    return _det_plan(case, env)
  if case.kind == 'ens':
    p = _ens_plan(case, env)
    if case.host:
      g = host_groups(case)
      return dataclasses.replace(p, launches=2 * g, groups=g)
    return p
  return _energy_plan(case)


# ---- float64 reference -----------------------------------------------------------
def point_values(case):
  """name -> [nfield, nrow, ncol] float64 point-wise terms of the public
  statistics (NaN where the kernel sees NaN)."""
  with np.errstate(invalid='ignore'):
    if case.kind == 'vector':
      du = case.fields('f') - case.fields('t')
      dv = case.fields('fv') - case.fields('tv')
      return {'vec': du * du + dv * dv}
    if case.kind == 'det':
      f, t = case.fields('f'), case.fields('t')
      d = f - t
      out = {'d2': d * d, 'ad': np.abs(d), 'd': d}
      if case.clim:
        c = case.fields('c')
        fa, ta = f - c, t - c
        out.update(fata=fa * ta, fa2=fa * fa, ta2=ta * ta)
      return out
    if case.kind == 'ens':
      x, t = case.fields('x'), case.fields('t')
      res = {k: [] for k in ('skill', 'spread', 'mse', 'var', 'deb')}
      for i in range(x.shape[0]):
        vals = _ens_point_np(x[i], t[i], case.skipna)
        for k, v in zip(res, vals):
          res[k].append(v)
      return {k: np.stack(v) for k, v in res.items()}
    x, t = case.fields('x'), case.fields('t')
    M = case.nmember
    out = {}
    for m in range(M):
      out[f'sk{m}'] = (x[:, m] - t) ** 2
      if m < M - 1:
        out[f'sp{m}'] = (x[:, m] - x[:, m + 1]) ** 2
    return out


def _ens_point_np(xs, ts, skipna):
  import warnings  # pylint: disable=import-outside-toplevel
  M = xs.shape[0]
  mean_fn = np.nanmean if skipna else np.mean
  with warnings.catch_warnings():
    warnings.simplefilter('ignore', RuntimeWarning)
    skill = mean_fn(np.abs(ts[None] - xs), axis=0)
    if M < 2:
      spread = np.zeros_like(ts)
    else:
      order = np.sort(xs, axis=0)
      rank = np.arange(1, M + 1, dtype=np.float64)[:, None, None]
      if skipna:
        n = (~np.isnan(xs)).sum(axis=0).astype(np.float64)
        spread = 2.0 * np.nansum((2 * rank - M - 1) * order, axis=0) / np.where(
            n > 0, n, np.nan) / (M - 1)
      else:
        spread = 2.0 * ((2 * rank - M - 1) * order).mean(axis=0) / (M - 1)
    xbar = mean_fn(xs, axis=0)
    mse = (ts - xbar) ** 2
    var = ((np.nanvar if skipna else np.var)(xs, axis=0, ddof=1) if M > 1
           else np.full_like(ts, np.nan))
    deb = mse - var / M
  return skill, spread, mse, var, deb


def select_fields(case, order):
  """The same case restricted to the fields `order` (in that order)."""
  return dataclasses.replace(case, offsets={k: v[np.asarray(order)]
                                            for k, v in case.offsets.items()})


def _wsum(W, v, skipna, zero_skip):
  """(sum W*v, sum W*[v valid]) per field and region: W [R, nrow, ncol],
  v [nfield, nrow, ncol] -> two [nfield, R] arrays."""
  nf, R = v.shape[0], W.shape[0]
  Wf = W.reshape(R, -1)
  vf = v.reshape(nf, -1)
  if not np.isnan(vf).any() and np.isfinite(vf).all():
    return vf @ Wf.T, np.broadcast_to(Wf.sum(axis=1), (nf, R)).copy()
  s = np.empty((nf, R))
  ws = np.empty((nf, R))
  with np.errstate(invalid='ignore'):
    for r in range(R):
      vr = np.where(Wf[r] > 0, vf, 0.0) if zero_skip else vf
      valid = ~np.isnan(vr)
      if skipna:
        s[:, r] = (np.where(valid, vr, 0.0) * Wf[r]).sum(axis=1)
        ws[:, r] = (valid * Wf[r]).sum(axis=1)
      else:
        s[:, r] = (vr * Wf[r]).sum(axis=1)
        ws[:, r] = Wf[r].sum()
  return s, ws


def reference(case, vals=None):
  """The raw output the header documents, in float64."""
  vals = point_values(case) if vals is None else vals
  W = case.dense_w()
  nf, R = case.nfield, case.nregion
  zs, sk = case.zero_skip, case.skipna
  if case.kind in ('det', 'vector'):
    out = np.zeros((nf, R, DET_NSTAT))
    if case.kind == 'vector':
      out[..., 0], out[..., 6] = _wsum(W, vals['vec'], sk, zs)
      return out
    names = ['d2', 'ad', 'd'] + (['fata', 'fa2', 'ta2'] if case.clim else [])
    cnt = {'d2': 6, 'fata': 7, 'fa2': 8, 'ta2': 9}
    for k, n in enumerate(names):
      s, ws = _wsum(W, vals[n], sk, zs)
      out[..., k] = s
      if n in cnt:
        out[..., cnt[n]] = ws
    return out
  if case.kind == 'ens':
    out = np.zeros((nf, R, ENS_NSTAT))
    for k, n in enumerate(('skill', 'spread', 'mse', 'var', 'deb')):
      out[..., k], out[..., 5 + k] = _wsum(W, vals[n], sk, zs)
    return out
  M = case.nmember
  out = np.zeros((nf, R, 4, M))
  for m in range(M):
    out[:, :, 0, m], out[:, :, 2, m] = _wsum(W, vals[f'sk{m}'], False, zs)
    if m < M - 1:
      out[:, :, 1, m], out[:, :, 3, m] = _wsum(W, vals[f'sp{m}'], False, zs)
  return out


def exact_slots(case):
  """Boolean mask over the last output axis / axes of the slots that are
  exact on this case (the rest: ens_bound)."""
  if case.kind != 'ens':
    return None
  m = np.ones(ENS_NSTAT, bool)
  m[[1, 3, 4]] = False
  if case.nmember & (case.nmember - 1):  # 1 / M is not a power of two
    m[[0, 2]] = False
  return m


def ens_bound(case, vals):
  """Bound on |kernel - reference| per (field, region, stat) for K2 / K2b
  slots that are not exact.  Per point the kernel forms each statistic in
  float32 from the members: the mean, 1 / M and 1 / (M - 1) carry a rounding
  each, and every sum over the members a rounding per term, so a point's
  error is at most (2 M + 8) u A^p, A = max(|t|, |x_m|) the point's scale,
  p = 1 for skill and spread and 2 for mse, var and debiased mse.  The
  float32 (row, segment) sum of n cells adds n u sum |wc val|, and the float64
  region sums are exact to 2^-50.  So |err| <= (2 M + 8 + n) u sum |W| (A^p +
  |val|), n the widest segment."""
  x, t = case.fields('x'), case.fields('t')
  with np.errstate(invalid='ignore'):
    A = np.nanmax(np.abs(np.concatenate([x, t[:, None]], axis=1)), axis=1)
  n = int(np.diff(case.seg_start).max())
  k = (2 * case.nmember + 8 + n) * U
  W = np.abs(case.dense_w())
  out = np.zeros((case.nfield, case.nregion, ENS_NSTAT))
  for j, (name, p) in enumerate((('skill', 1), ('spread', 1), ('mse', 2),
                                 ('var', 2), ('deb', 2))):
    mag = np.nan_to_num(A ** p + np.abs(vals[name]), nan=0.0, posinf=0.0)
    out[..., j] = k * (mag.reshape(case.nfield, -1) @ W.reshape(case.nregion, -1).T)
  return out


# ---- bit budget ------------------------------------------------------------------
def _lsb_exp(a):
  """Exponent of the lowest set bit of every element (+inf for 0 / NaN)."""
  a = np.abs(np.asarray(a, np.float64))
  ok = np.isfinite(a) & (a != 0)
  m, e = np.frexp(np.where(ok, a, 1.0))
  im = (m * 2.0 ** 53).astype(np.int64)
  low = im & -im
  tz = np.log2(low.astype(np.float64))
  return np.where(ok, e - 53 + tz, np.inf)


def _span(terms, axis):
  """log2(sum |terms|) - lowest set bit over `axis` (-inf when all zero)."""
  a = np.nan_to_num(np.abs(terms), nan=0.0, posinf=0.0)
  tot = a.sum(axis=axis)
  lsb = _lsb_exp(np.where(np.isfinite(terms), terms, 0)).min(axis=axis)
  with np.errstate(divide='ignore', invalid='ignore'):
    return np.where(tot > 0, np.log2(np.where(tot > 0, tot, 1)) - lsb, -np.inf)


def _exact_terms(case, vals):
  count = np.ones_like(next(iter(vals.values())))
  if case.kind == 'ens':
    keep = [n for n, e in zip(('skill', 'spread', 'mse', 'var', 'deb'),
                              exact_slots(case)[:5]) if e]
    vals = {k: vals[k] for k in keep}
  return dict(vals, count=count)


def bit_budget(case, env=None):
  """Worst-case span in bits of every accumulator the planned path uses:
  'f32_rowseg' the float32 (row, segment) sums (LDG, TMA half rows, pair /
  scalar K2, K3), 'f32_band' TMA-seg's band accumulator and its per-region
  dump over at most 16 tiles of a warp pair (bounded by any 8 * CW
  consecutive rows of one half row), 'f64_region' the float64 region sums.
  Returns {name: bits}; exactness needs <= 24 / 53."""
  p = plan(case, env)
  vals = _exact_terms(case, point_values(case))
  W = case.dense_w()
  wc = np.ones((case.nrow, case.ncol))
  if case.col_w is not None:
    wc = wc * case.col_w.astype(np.float64)[None]
  if case.cell_w is not None:
    wc = wc * case.cell_w.astype(np.float64)
  out = {'f64_region': -np.inf}
  f32 = case.dtype == np.float32 and p.path != 'big'
  if f32:
    out['f32_rowseg'] = -np.inf
  if p.path == 'tma_seg':
    out['f32_band'] = -np.inf
  for v in vals.values():
    v = np.where(np.isnan(v) | np.isinf(v), 0.0, v)
    for r in range(case.nregion):
      out['f64_region'] = max(out['f64_region'],
                              np.max(_span((v * W[r]).reshape(v.shape[0], -1), 1)))
    if f32 and p.path != 'tma_seg':
      tv = v * wc
      for k in range(case.nseg):
        a, b = case.seg_start[k], case.seg_start[k + 1]
        out['f32_rowseg'] = max(out['f32_rowseg'], np.max(_span(tv[..., a:b], 2)))
    if p.path == 'tma_seg':
      L = 8 * p.cw
      h = (case.ncol + 1) // 2
      for r in range(-1, case.nregion):
        # r = -1: the band accumulator itself, row_c * part
        ww = (np.abs(case.row_w).max(axis=0)[:, None] * np.ones(case.ncol)
              if r < 0 else W[r])
        tv = v * ww
        for a, b in ((0, h), (h, case.ncol)):
          rowsum = np.abs(tv[..., a:b]).sum(axis=2)  # [nf, nrow]
          cs = np.concatenate([np.zeros((rowsum.shape[0], 1)),
                               np.cumsum(rowsum, axis=1)], axis=1)
          win = cs[:, L:] - cs[:, :-L] if case.nrow > L else cs[:, -1:]
          tot = win.max()
          lsb = _lsb_exp(tv[..., a:b]).min()
          if tot > 0:
            out['f32_band'] = max(out['f32_band'], np.log2(tot) - lsb)
  return out


# ---- the exact family ------------------------------------------------------------
def _det_case(name, rs, *, nrow, ncol, nfield=3, row_stride=None, nregion=1,
              seg_start=None, clim=False, skipna=False, dtype=np.float32,
              col_w=False, cell_w=False, zero_skip=True, align=4, shift=0,
              row_w=None, nan_frac=0.0, env=({},), covers=(), kind='det',
              host=False, stage_mb=0, neg=False, jmax=3, seg_w=None):
  seg_start = [0, ncol] if seg_start is None else list(seg_start)
  rw, ss, sw = _weights(rs, nrow, ncol, nregion, seg_start, neg=neg, jmax=jmax,
                        row_zero=0.25 if zero_skip else 0.1)
  if row_w is not None:
    rw = row_w
  if seg_w is not None:
    sw = seg_w
  case = Case(name, kind, nrow, ncol, row_stride or ncol, rw, ss, sw,
              zero_skip=zero_skip, skipna=skipna, dtype=dtype, clim=clim,
              env=env, covers=covers, host=host, stage_mb=stage_mb)
  if col_w:
    case.col_w = _pow2(rs, ncol, 2, 0.1 if zero_skip else 0.0).astype(np.float32)
  if cell_w:
    case.cell_w = _pow2(rs, (nrow, ncol), 2, 0.1 if zero_skip else 0.0).astype(
        np.float32)
  case._align, case._shift = align, shift  # pylint: disable=protected-access
  names = (['f', 't', 'fv', 'tv'] if kind == 'vector' else
           ['f', 't'] + (['c'] if clim else []))
  values = {n: _grid(rs, (nfield, nrow, ncol)) for n in names}
  # NaN in every operand, at different cells, so that each skipna count
  # slot (d, fa * ta, fa, ta valid) differs from the others
  nan_cells = ({n: rs.rand(nfield, nrow, ncol) < nan_frac * (1.0 if k == 0 else 0.5)
                for k, n in enumerate(names)} if nan_frac else None)
  return _finish(case, rs, values, nan_cells)


def _ens_case(name, rs, *, M, nrow, ncol, nfield=2, kind='ens', row_stride=None,
              nregion=1, seg_start=None, skipna=False, col_w=False,
              cell_w=False, ms_extra=0, shift=0, align=4, env=({},),
              covers=(), host=False, stage_mb=0, nan_truth=0.0,
              zero_skip=True, step=0.5):
  seg_start = [0, ncol] if seg_start is None else list(seg_start)
  rw, ss, sw = _weights(rs, nrow, ncol, nregion, seg_start)
  rs_ = row_stride or ncol
  span = (nrow - 1) * rs_ + ncol
  ms = (span + 4) // 4 * 4 + ms_extra  # NaN gap between members
  case = Case(name, kind, nrow, ncol, rs_, rw, ss, sw, zero_skip=zero_skip,
              skipna=skipna, nmember=M, member_stride=ms, env=env,
              covers=covers, host=host, stage_mb=stage_mb)
  if col_w:
    case.col_w = _pow2(rs, ncol, 2, 0.1).astype(np.float32)
  if cell_w:
    case.cell_w = _pow2(rs, (nrow, ncol), 2, 0.1).astype(np.float32)
  case._align, case._shift = align, shift  # pylint: disable=protected-access
  x = _grid(rs, (nfield, M, nrow, ncol), step)
  t = _grid(rs, (nfield, nrow, ncol), step)
  if nan_truth:
    t = np.where(rs.rand(*t.shape) < nan_truth, np.nan, t)
  return _finish(case, rs, {'x': x, 't': t})


def _det_env(tma_like):
  return ({}, {'WB2_DET_PATH': 'ldg'}) if tma_like else ({},)


def exact_cases():
  """The exact family: name -> Case (seeded, deterministic)."""
  rs = np.random.RandomState(20261015)
  cs = []
  tma_env = _det_env(True)
  seg_env = ({}, {'WB2_DET_PATH': 'ldg'})
  # ---- K1 TMA, one segment -------------------------------------------------------
  for nrow, ncol, nfield in ((1, 128, 5), (2, 132, 3), (3, 1440, 2), (181, 128, 2)):
    for clim in (False, True):
      for skipna in (False, True):
        cs.append(_det_case(
            f'k1_tma_r{nrow}_c{ncol}_{"clim" if clim else "plain"}_sk{int(skipna)}',
            rs, nrow=nrow, ncol=ncol, nfield=nfield, clim=clim, skipna=skipna,
            nregion=(1, 31, 32, 3)[(nrow + ncol) % 4], nan_frac=0.05 * skipna,
            env=tma_env, covers=('k1_tma_plain' if not clim else 'k1_tma_clim',)))
  cs.append(_det_case('k1_tma_r31', rs, nrow=5, ncol=256, nfield=20, nregion=31,
                      env=tma_env, covers=('k1_tma_nregion31',)))
  cs.append(_det_case('k1_tma_r32_grid', rs, nrow=7, ncol=128, nfield=18,
                      nregion=32, clim=True, env=tma_env,
                      covers=('k1_tma_nregion32', 'tma_ntiles_lt_sms')))
  cs.append(_det_case('k1_tma_uneven_grid', rs, nrow=3, ncol=128, nfield=100,
                      nregion=2, skipna=True, nan_frac=0.03, env=tma_env,
                      covers=('tma_ntiles_mod_ncta', 'tma_many_fields_per_cta')))
  cs.append(_det_case('k1_tma_r1', rs, nrow=181, ncol=128, nfield=1, nregion=1,
                      env=tma_env, covers=('k1_tma_nregion1',)))
  cs.append(_det_case('k1_tma_stage_fallback', rs, nrow=2, ncol=9600, nfield=2,
                      clim=True, nregion=2, covers=('k1_tma_stage_fallback',)))
  # ---- K1 TMA-seg ----------------------------------------------------------------
  for nreg in (8, 9, 16, 17, 32):
    for skipna in (False, True):
      ss = [0, 20, 44, 64, 100, 128]
      cs.append(_det_case(
          f'k1_seg_r{nreg}_sk{int(skipna)}', rs, nrow=24, ncol=128, nfield=3,
          nregion=nreg, seg_start=ss, skipna=skipna, nan_frac=0.04 * skipna,
          row_w=_banded_row_w(rs, 24, nreg, 5), env=seg_env,
          covers=('k1_seg_chunks',)))
  cs.append(_det_case('k1_seg_128_bands', rs, nrow=128, ncol=128, nfield=2,
                      nregion=4, seg_start=[0, 64, 128],
                      row_w=_banded_row_w(rs, 128, 4, 128, 2), env=seg_env,
                      covers=('k1_seg_128_bands',)))
  cs.append(_det_case('k1_seg_129_bands', rs, nrow=129, ncol=128, nfield=2,
                      nregion=4, seg_start=[0, 64, 128],
                      row_w=_banded_row_w(rs, 129, 4, 129, 2),
                      covers=('k1_seg_129_bands_ldg',)))
  ss = np.unique(np.concatenate([[0, 128], np.arange(1, 80, 2)])).astype(np.int32)
  cs.append(_det_case('k1_seg_second_round', rs, nrow=6, ncol=128, nfield=2,
                      nregion=17, seg_start=ss, env=seg_env,
                      covers=('k1_seg_second_round',)))
  cs.append(_det_case('k1_seg_clim_skipna', rs, nrow=20, ncol=128, nfield=3,
                      nregion=12, seg_start=[0, 9, 64, 100, 128], clim=True,
                      skipna=True, nan_frac=0.06,
                      row_w=_banded_row_w(rs, 20, 12, 4), env=seg_env,
                      covers=('k1_seg_chunks', 'k1_seg_clim_skipna')))
  ss = np.concatenate([np.arange(0, 101), [256]]).astype(np.int32)
  cs.append(_det_case('k1_seg_too_many_spans', rs, nrow=4, ncol=256, nfield=2,
                      nregion=2, seg_start=ss, covers=('k1_seg_spans_ldg',)))
  rw = _banded_row_w(rs, 32, 3, 4)
  rw[:, 5:9] = 0.0  # rows outside every region: row_c == 0
  rw[1, 20:32] = 0.0  # a band where region 1's pattern is 0, others not
  rw[0, 20:32] = np.where(rw[0, 20:32] == 0, 0.5, rw[0, 20:32])
  cs.append(_det_case('k1_seg_zero_rows', rs, nrow=32, ncol=256, nfield=2,
                      nregion=3, seg_start=[0, 40, 160, 256], row_w=rw,
                      clim=True, env=seg_env,
                      covers=('k1_seg_row_c_zero', 'k1_seg_zero_pattern')))
  # ---- K1 LDG --------------------------------------------------------------------
  for r in range(4):
    ss = [0, 8 + r, 17 + r, 18 + r, 20 + r, 23 + r, 64 + r, 200]
    cs.append(_det_case(f'k1_ldg_vec4_res{r}', rs, nrow=5, ncol=200, nfield=2,
                        nregion=3, seg_start=ss, col_w=True,
                        covers=('k1_ldg_residues', 'k1_ldg_short_segments')))
  cs.append(_det_case('k1_ldg_odd_offsets', rs, nrow=6, ncol=133, nfield=3,
                      row_stride=141, nregion=5, seg_start=[0, 7, 70, 133],
                      shift=1, skipna=True, clim=True, nan_frac=0.05,
                      covers=('k1_ldg_vec1',)))
  cs.append(_det_case('k1_ldg_f64_vec2', rs, nrow=9, ncol=130, nfield=3,
                      dtype=np.float64, nregion=4, seg_start=[0, 3, 65, 130],
                      clim=True, align=2, covers=('k1_ldg_f64_vec2',)))
  cs.append(_det_case('k1_ldg_f64_vec1', rs, nrow=9, ncol=131, nfield=3,
                      dtype=np.float64, nregion=4, seg_start=[0, 66, 131],
                      skipna=True, nan_frac=0.05, shift=1,
                      covers=('k1_ldg_f64_vec1',)))
  cs.append(_det_case('k1_ldg_col_w', rs, nrow=7, ncol=128, nfield=2,
                      nregion=3, col_w=True, clim=True, covers=('k1_ldg_col_w',)))
  cs.append(_det_case('k1_ldg_cell_w', rs, nrow=7, ncol=128, nfield=2,
                      nregion=3, cell_w=True, skipna=True, nan_frac=0.05,
                      covers=('k1_ldg_cell_w',)))
  cs.append(_det_case('k1_ldg_col_and_cell_w', rs, nrow=7, ncol=132, nfield=2,
                      nregion=3, col_w=True, cell_w=True,
                      seg_start=[0, 33, 99, 132], clim=True,
                      covers=('k1_ldg_col_and_cell_w',)))
  cs.append(_det_case('k1_row_stride', rs, nrow=6, ncol=128, row_stride=148,
                      nfield=3, nregion=2, clim=True, env=tma_env,
                      covers=('row_stride_gt_ncol',)))
  cs.append(_det_case('k1_ldg_one_field_halved', rs, nrow=181, ncol=40,
                      nfield=1, nregion=3, seg_start=[0, 12, 40],
                      covers=('k1_ldg_halved_rows',)))
  cs.append(_det_case('k1_vector', rs, nrow=6, ncol=64, nfield=3, nregion=3,
                      seg_start=[0, 21, 64], kind='vector', skipna=True,
                      covers=('k1_vector',)))
  cs.append(_det_case('k1_negative_weights', rs, nrow=6, ncol=128, nfield=2,
                      nregion=3, zero_skip=False, neg=True, env=tma_env,
                      covers=('negative_weights',)))
  cs.append(_det_case('k1_negative_weights_seg', rs, nrow=6, ncol=128, nfield=2,
                      nregion=3, zero_skip=False, neg=True,
                      seg_start=[0, 50, 128], env=seg_env,
                      covers=('negative_weights',)))
  # ---- K2 ------------------------------------------------------------------------
  pair_env = ({}, {'WB2_ENS_PATH': 'scalar'},
              {'WB2_ENS_PATH': 'scalar', 'WB2_ENS_SORT': 'exact'})
  for M in (8, 16, 32, 64):
    cs.append(_ens_case(f'k2_pair_m{M}', rs, M=M, nrow=5, ncol=64, nregion=3,
                        env=pair_env,
                        covers=('k2_pair', 'k2_twin_and_exact_sort',
                                'k2_scalar_exact_sort')))
  for M in (6, 33):
    cs.append(_ens_case(f'k2_scalar_m{M}', rs, M=M, nrow=4, ncol=40, nregion=2,
                        seg_start=[0, 17, 40], covers=('k2_inexact_mp',)))
  cs.append(_ens_case('k2_skipna', rs, M=16, nrow=5, ncol=48, nregion=3,
                      skipna=True, nan_truth=0.1, covers=('k2_skipna',)))
  cs.append(_ens_case('k2_occ', rs, M=10, nrow=6, ncol=64, nregion=2,
                      seg_start=[0, 30, 64]))
  cs.append(_ens_case('k2_weighted', rs, M=8, nrow=5, ncol=36, nregion=4,
                      seg_start=[0, 5, 6, 36], col_w=True, cell_w=True,
                      covers=('k2_weighted',)))
  cs.append(_ens_case('k2_odd_ncol', rs, M=8, nrow=3, ncol=63,
                      covers=('k2_pair_odd_ncol',)))
  cs.append(_ens_case('k2_odd_row_stride', rs, M=8, nrow=3, ncol=64,
                      row_stride=67, covers=('k2_pair_odd_row_stride',)))
  cs.append(_ens_case('k2_odd_member_stride', rs, M=8, nrow=3, ncol=64,
                      ms_extra=1, covers=('k2_pair_odd_member_stride',)))
  cs.append(_ens_case('k2_odd_offset', rs, M=8, nrow=3, ncol=64, shift=1,
                      covers=('k2_pair_odd_offset',)))
  # ---- K2b -----------------------------------------------------------------------
  cs.append(_ens_case('k2b_m65', rs, M=65, nrow=3, ncol=45, nregion=3,
                      seg_start=[0, 10, 33, 45], covers=('k2b',)))
  cs.append(_ens_case('k2b_m128', rs, M=128, nrow=2, ncol=70, nregion=2,
                      seg_start=[0, 31, 70], cell_w=True, skipna=True,
                      nan_truth=0.1, covers=('k2b', 'k2b_partial_tile')))
  # ---- K3 ------------------------------------------------------------------------
  for M in (1, 3, 4, 5, 17, 64):
    cs.append(_ens_case(f'k3_vec4_m{M}', rs, M=M, nrow=3, ncol=64, nregion=2,
                        kind='energy', seg_start=[0, 32, 64],
                        covers=('k3_vec4', 'k3_gs')))
  cs.append(_ens_case('k3_scalar_boundary', rs, M=5, nrow=3, ncol=64,
                      nregion=2, kind='energy', seg_start=[0, 30, 64],
                      covers=('k3_scalar_boundary',)))
  cs.append(_ens_case('k3_scalar_member_stride', rs, M=8, nrow=3, ncol=64,
                      kind='energy', ms_extra=1,
                      covers=('k3_scalar_member_stride',)))
  cs.append(_ens_case('k3_weighted', rs, M=9, nrow=4, ncol=64, nregion=3,
                      kind='energy', col_w=True, cell_w=True,
                      seg_start=[0, 16, 64], covers=('k3_weighted',)))
  # ---- host entries ----------------------------------------------------------------
  cs.append(_det_case('host_det_cell_w_stride', rs, nrow=6, ncol=128,
                      row_stride=136, nfield=4, nregion=3, cell_w=True,
                      clim=True, host=True, covers=('host_det',)))
  cs.append(_det_case('host_det_tma_groups', rs, nrow=181, ncol=360, nfield=8,
                      nregion=2, host=True, stage_mb=1,
                      covers=('host_det', 'host_groups')))
  cs.append(_ens_case('host_ens_groups', rs, M=8, nrow=91, ncol=180,
                      row_stride=184, nfield=3, nregion=2, cell_w=True,
                      host=True, stage_mb=1, covers=('host_ens', 'host_groups')))
  return {c.name: c for c in cs}


# Each coverage item: predicate over (case, plan of the default env, plans of
# every env variant).  The CPU test asserts every item is reached.
def nan_per_region(c):
  """Some field's reference holds NaN / Inf in some but not all regions."""
  ref = reference(c)
  bad = ~np.isfinite(ref).reshape(ref.shape[0], ref.shape[1], -1).all(axis=2)
  return bool((bad.any(axis=1) & ~bad.all(axis=1)).any())


def _any(pred):
  return lambda c, p, ps: any(pred(c, q) for q in ps)


COVERAGE = {
    'k1_tma_plain': lambda c, p, ps: p.path == 'tma' and not c.clim,
    'k1_tma_clim': lambda c, p, ps: p.path == 'tma' and c.clim,
    'k1_tma_nregion1': lambda c, p, ps: p.path == 'tma' and c.nregion == 1,
    'k1_tma_nregion31': lambda c, p, ps: p.path == 'tma' and c.nregion == 31,
    'k1_tma_nregion32': lambda c, p, ps: p.path == 'tma' and c.nregion == 32,
    'tma_ntiles_lt_sms': lambda c, p, ps: (p.path == 'tma' and
                                           c.nrow * c.nfield < NUM_SMS),
    'tma_ntiles_mod_ncta': lambda c, p, ps: (p.path == 'tma' and
                                             c.nrow * c.nfield > NUM_SMS and
                                             (c.nrow * c.nfield) % NUM_SMS != 0),
    'tma_many_fields_per_cta': lambda c, p, ps: (p.path == 'tma' and c.nrow < 4 and
                                                 c.nrow * c.nfield > NUM_SMS),
    'k1_tma_stage_fallback': lambda c, p, ps: (p.path == 'ldg' and c.clim and
                                               c.nseg == 1 and c.ncol * 4 >= 512),
    'k1_seg_chunks': lambda c, p, ps: p.path == 'tma_seg',
    'k1_seg_128_bands': lambda c, p, ps: (p.path == 'tma_seg' and
                                          max(p.bands) == 128),
    'k1_seg_129_bands_ldg': lambda c, p, ps: (p.path == 'ldg' and c.nseg > 1 and
                                              seg_bands(c.row_w, 16) is None),
    'k1_seg_second_round': lambda c, p, ps: (p.path == 'tma_seg' and
                                             max(p.rounds) == 2 and
                                             p.launches != 2),
    'k1_seg_clim_skipna': lambda c, p, ps: (p.path == 'tma_seg' and c.clim and
                                            c.skipna and p.chunks > 1),
    'k1_seg_spans_ldg': lambda c, p, ps: (p.path == 'ldg' and
                                          seg_spans(c.ncol, c.seg_start) is None),
    'k1_seg_row_c_zero': lambda c, p, ps: (
        p.path == 'tma_seg' and c.zero_skip and
        (np.abs(c.row_w).max(axis=0) == 0).any()),
    'k1_seg_zero_pattern': lambda c, p, ps: (
        p.path == 'tma_seg' and
        ((c.row_w == 0) & (np.abs(c.row_w).max(axis=0) > 0)[None]).any()),
    'k1_ldg_residues': lambda c, p, ps: p.path == 'ldg' and p.vec == 4,
    'k1_ldg_short_segments': lambda c, p, ps: (
        p.path == 'ldg' and p.vec == 4 and
        {1, 2, 3} <= set(np.diff(c.seg_start).tolist())),
    'k1_ldg_vec1': lambda c, p, ps: (p.path == 'ldg' and p.vec == 1 and
                                     c.dtype == np.float32),
    'k1_ldg_f64_vec2': lambda c, p, ps: c.dtype == np.float64 and p.vec == 2,
    'k1_ldg_f64_vec1': lambda c, p, ps: c.dtype == np.float64 and p.vec == 1,
    'k1_ldg_col_w': lambda c, p, ps: c.col_w is not None and c.cell_w is None,
    'k1_ldg_cell_w': lambda c, p, ps: c.cell_w is not None and c.col_w is None,
    'k1_ldg_col_and_cell_w': lambda c, p, ps: (c.cell_w is not None and
                                               c.col_w is not None),
    'row_stride_gt_ncol': lambda c, p, ps: c.row_stride > c.ncol,
    'k1_ldg_halved_rows': lambda c, p, ps: (
        p.path == 'ldg' and c.nfield == 1 and p.rows_per_block < 32 and
        c.nrow % p.rows_per_block != 0),
    'k1_vector': lambda c, p, ps: c.kind == 'vector',
    'negative_weights': lambda c, p, ps: (not c.zero_skip and
                                          (c.dense_w() < 0).any()),
    'k2_pair': lambda c, p, ps: p.path == 'pair' and c.nmember in (8, 16, 32, 64),
    'k2_twin_and_exact_sort': _any(lambda c, q: q.path == 'twin'),
    'k2_scalar_exact_sort': _any(lambda c, q: q.path == 'scalar' and
                                 c.nmember in (8, 16, 32, 64)),
    'k2_inexact_mp': lambda c, p, ps: p.path == 'scalar' and c.nmember in (6, 33),
    'k2_skipna': lambda c, p, ps: p.path == 'scalar' and c.skipna,
    'k2_weighted': lambda c, p, ps: (c.kind == 'ens' and c.nseg > 1 and
                                     c.col_w is not None and c.cell_w is not None),
    'k2_pair_odd_ncol': lambda c, p, ps: p.path == 'twin' and c.ncol % 2,
    'k2_pair_odd_row_stride': lambda c, p, ps: p.path == 'twin' and c.row_stride % 2,
    'k2_pair_odd_member_stride': lambda c, p, ps: (p.path == 'twin' and
                                                   c.member_stride % 2),
    'k2_pair_odd_offset': lambda c, p, ps: (p.path == 'twin' and
                                            (c.offsets['x'] % 2).any()),
    'k2b': lambda c, p, ps: p.path == 'big' and c.nseg > 1,
    'k2b_partial_tile': lambda c, p, ps: (p.path == 'big' and c.ncol % 32 and
                                          c.cell_w is not None and c.skipna),
    'k3_vec4': lambda c, p, ps: p.path == 'energy' and p.vec4,
    'k3_gs': lambda c, p, ps: (p.path == 'energy' and
                               p.gs == (4 if c.nmember <= 4 else 8)),
    'k3_scalar_boundary': lambda c, p, ps: (p.path == 'energy' and not p.vec4 and
                                            (c.seg_start % 4).any()),
    'k3_scalar_member_stride': lambda c, p, ps: (p.path == 'energy' and
                                                 not p.vec4 and c.member_stride % 2),
    'k3_weighted': lambda c, p, ps: (p.path == 'energy' and c.cell_w is not None and
                                     c.col_w is not None),
    'host_det': lambda c, p, ps: c.host and c.kind == 'det',
    'host_ens': lambda c, p, ps: c.host and c.kind == 'ens',
    'host_groups': lambda c, p, ps: c.host and p.groups > 1,
}


# ---- realistic family ------------------------------------------------------------
def official_regions(lsm):
  """The 16 regions of the reference's scripts/evaluate.py (the same list as
  test_official_configs.predefined_regions)."""
  from weatherbench2_b200 import regions as R  # pylint: disable=import-outside-toplevel
  S = R.SliceRegion
  et = [slice(None, -20), slice(20, None)]
  return [
      S(), S(lat_slice=slice(-20, 20)), S(lat_slice=et),
      S(lat_slice=slice(20, None)), S(lat_slice=slice(None, -20)),
      S(lat_slice=slice(35, 75), lon_slice=[slice(360 - 12.5, None), slice(0, 42.5)]),
      S(lat_slice=slice(25, 60), lon_slice=slice(360 - 120, 360 - 75)),
      S(lat_slice=slice(25, 65), lon_slice=slice(360 - 70, 360 - 10)),
      S(lat_slice=slice(25, 60), lon_slice=slice(145, 360 - 130)),
      S(lat_slice=slice(25, 60), lon_slice=slice(102.5, 150)),
      S(lat_slice=slice(-45, -12.5), lon_slice=slice(120, 175)),
      S(lat_slice=slice(60, 90)), S(lat_slice=slice(-90, -60)),
      R.LandRegion(lsm),
      R.CombinedRegion([S(lat_slice=et), R.LandRegion(lsm)]),
      R.CombinedRegion([S(lat_slice=slice(-20, 20)), R.LandRegion(lsm)]),
  ]


def fractional_lsm(nlat, nlon, seed=3):
  """A smooth land fraction in [0, 1] with exact 0 and 1 areas (LandRegion's
  fractional cell weights)."""
  rs = np.random.RandomState(seed)
  la = np.linspace(0, np.pi, nlat)[:, None]
  lo = np.linspace(0, 2 * np.pi, nlon, endpoint=False)[None]
  v = np.sin(3 * lo + rs.rand()) * np.cos(2 * la) + 0.3 * rs.randn(nlat, nlon)
  return np.clip(v, 0.0, 1.0).astype(np.float32)


def realistic_cases(ctx, which=None):
  """The realistic family (not exact): one Case per launch group that
  _spatial.build_weights makes for the 16 official regions on a 0.25 / 1
  degree grid, cosine latitude weights, a fractional land mask, both layouts;
  float32 inputs from a normal distribution.  ctx uploads the cell weights
  (a FakeContext keeps them in host memory)."""
  from weatherbench2_b200 import _spatial as sp  # pylint: disable=import-outside-toplevel
  out = []
  for k, (name, nlat, nlon, layout, nfield, regs, kind) in enumerate(REALISTIC):
    if which is not None and name not in which:
      continue
    rs = np.random.RandomState(100 + k)
    lat = np.linspace(-90, 90, nlat)
    lon = np.linspace(0, 360, nlon, endpoint=False)
    lsm = fractional_lsm(nlat, nlon)
    regions = official_regions(lsm)
    if regs == 'land':
      regions = regions[13:]
    nrow, ncol = (nlat, nlon) if layout == 'lat_lon' else (nlon, nlat)
    for g, (_, spec) in enumerate(sp.build_weights(ctx, lat, lon, regions,
                                                   layout, ncol)):
      cell = (None if spec.cell_w_dev is None else
              ctx.from_device(spec.cell_w_dev, (nrow, ncol), np.float32))
      case = Case(f'{name}_g{g}', kind, nrow, ncol, ncol, spec.row_w,
                  spec.seg_start, spec.seg_w, spec.col_w, cell,
                  zero_skip=spec.zero_skip, clim=regs == 'land',
                  exact=False, cell_w_dev=spec.cell_w_dev)
      if kind == 'ens':
        case.nmember = 10
        case.member_stride = nrow * ncol + 4
        vals = {'x': rs.randn(nfield, 10, nrow, ncol),
                't': rs.randn(nfield, nrow, ncol)}
      else:
        names = ['f', 't'] + (['c'] if case.clim else [])
        vals = {n: rs.randn(nfield, nrow, ncol) * 100 + 5000 * (n == 'c')
                for n in names}
        if case.clim:
          vals['f'] = vals['f'] + 5000
          vals['t'] = vals['t'] + 5000
      out.append(_finish(case, rs, vals, sentinel_in_zero=False, poison=False))
  return out


REALISTIC = (
    # name, nlat, nlon, layout, nfield, regions ('official' | 'land'), kind
    ('real_181x360_official', 181, 360, 'lat_lon', 3, 'official', 'det'),
    ('real_181x360_lonlat', 181, 360, 'lon_lat', 3, 'official', 'det'),
    ('real_181x360_clim_land', 181, 360, 'lat_lon', 2, 'land', 'det'),
    ('real_721x1440_official', 721, 1440, 'lat_lon', 1, 'official', 'det'),
    ('real_181x360_ens', 181, 360, 'lat_lon', 2, 'official', 'ens'),
)


def many_field_cases():
  """Launches with many fields, for the field-order / nfield-prefix test and
  the TMA scratch size: ncta * 8 warps * maxslots * nregion * 80 B of
  partials (nrow = 1, 20 000 fields, 32 regions: about 413 MB for a 51 MB
  output)."""
  rs = np.random.RandomState(7)
  cs = [
      _det_case('k1_tma_scratch', rs, nrow=1, ncol=128, nfield=20000,
                nregion=32),
      _det_case('k1_seg_many', rs, nrow=2, ncol=128, nfield=140, nregion=17,
                seg_start=[0, 24, 72, 128], clim=True),
      _det_case('k1_ldg_many', rs, nrow=3, ncol=72, nfield=140, nregion=3,
                seg_start=[0, 5, 72], skipna=True, nan_frac=0.05),
      _ens_case('k2_pair_many', rs, M=8, nrow=2, ncol=64, nfield=140,
                nregion=3),
      _ens_case('k3_many', rs, M=5, nrow=2, ncol=64, nfield=140, nregion=3,
                kind='energy'),
  ]
  return {c.name: c for c in cs}

"""TEST INFRASTRUCTURE: seeded raw-ABI cases for the three entries of
`csrc/threshold_metrics.cu` (wb2_ens_threshold_metrics, wb2_ens_threshold_maps,
wb2_gaussian_metrics), their float64 interpretation through the oracle, and a
NumPy model of the Gaussian kernel's float32 `z` with the error bounds the
GPU tests hold the kernel to.

A point-wise case holds one grid cell per field: the reduction entries run on
a 1 x 1 geometry with `off_*[i]` pointing at cell i, so each output is one
cell's score times weight 1; the maps entry runs the same cells as one
nrow x ncol map (cell c on lane c % 32 of CTA c // 128).  Members sit either
in the usual [member][field][cell] layout (`member_stride` = number of cells)
or interleaved per field ([field][member][cell], `member_stride` = 1)."""
from __future__ import annotations

import dataclasses
from fractions import Fraction
from typing import Optional

import numpy as np
from scipy import special, stats

from oracle import wb2_oracle as orc
from weatherbench2_b200 import _lib

F32, F64 = np.float32, np.float64
FLT_MAX = float(np.finfo(F32).max)
U = 2.0 ** -24                      # unit roundoff of float32
TAIL_SWITCH = float(F32(1e-7))      # the kernel's float32 / float64 switch
SATURATION = 2.0 ** -54             # 1 - tail rounds to 1 in float64 below
ERFC_UNDERFLOW = 709.782712893384   # scipy's erfc(a) is 0 once a^2 exceeds it
MAP_THREADS = 128                   # kThrThreads: cells per CTA of the maps


def down(v):
  return np.nextafter(F32(v), F32(-np.inf))


def up(v):
  return np.nextafter(F32(v), F32(np.inf))


def bracket(thr) -> tuple[np.ndarray, np.ndarray]:
  """float32 (lo, hi) = (round down, round up) of float64 thresholds."""
  thr = np.asarray(thr, F64)
  with np.errstate(over='ignore', invalid='ignore'):
    near = thr.astype(F32)
    nd = near.astype(F64)
    lo = np.where(nd > thr, np.nextafter(near, F32(-np.inf)), near)
    hi = np.where(nd < thr, np.nextafter(near, F32(np.inf)), near)
  return lo.astype(F32), hi.astype(F32)


def gauss_threshold(mean, std, z) -> np.ndarray:
  """thr = mean + z * std with two float64 roundings: [nq][ncell]."""
  mean = np.asarray(mean, F32).astype(F64)
  std = np.asarray(std, F32).astype(F64)
  with np.errstate(invalid='ignore', over='ignore'):
    return mean[None] + np.asarray(z, F64)[:, None] * std[None]


def fma_single_rounding(mean, std, z) -> float:
  """round(z * std + mean) with one rounding, exactly (Fraction)."""
  return float(Fraction(float(z)) * Fraction(float(std)) +
               Fraction(float(mean)))


# ---------------------------------------------------------------------------
# Cases
# ---------------------------------------------------------------------------
@dataclasses.dataclass
class Case:
  """One raw-ABI case; `ncell` cells, each its own field."""
  name: str
  kind: str                       # 'ens' or 'gauss'
  t: np.ndarray                   # float32 [ncell]
  nq: int
  thr_a: Optional[np.ndarray]     # field form [nq][ncell]; Gaussian form mean [ncell]
  thr_b: Optional[np.ndarray] = None   # Gaussian form: climatological std [ncell]
  z: Optional[np.ndarray] = None       # Gaussian form: [nq]
  members: Optional[np.ndarray] = None  # ens: float32 [M][ncell]
  interleaved: bool = False       # ens: members stored [cell][member]
  mean: Optional[np.ndarray] = None     # gauss: forecast mean [ncell]
  std: Optional[np.ndarray] = None      # gauss: forecast std [ncell]

  @property
  def ncell(self) -> int:
    return self.t.size

  @property
  def nmember(self) -> int:
    return self.members.shape[0]

  # -- raw arrays and arguments -------------------------------------------------
  def x_buffer(self) -> np.ndarray:
    m = self.members.T if self.interleaved else self.members
    return np.ascontiguousarray(m, F32).reshape(-1)

  def member_stride(self) -> int:
    return 1 if self.interleaved else self.ncell

  def off_x(self) -> np.ndarray:
    c = np.arange(self.ncell, dtype=np.int64)
    return c * self.nmember if self.interleaved else c

  def thr_buffers(self):
    """(thr_a buffer, thr_b buffer or None), float32."""
    a = np.ascontiguousarray(self.thr_a, F32).reshape(-1)
    b = None if self.thr_b is None else np.ascontiguousarray(self.thr_b, F32)
    return a, b

  def off_thr(self):
    """Point-wise (off_a, off_b): one field per cell."""
    c = np.arange(self.ncell, dtype=np.int64)
    if self.thr_b is not None:
      return c, c.copy()
    return (np.arange(self.nq, dtype=np.int64)[:, None] * self.ncell +
            c[None]).reshape(-1), None

  # -- float64 interpretation -----------------------------------------------------
  def thresholds(self) -> np.ndarray:
    """float64 thresholds [nq][ncell] as the kernel forms them."""
    if self.nq == 0:
      return np.zeros((0, self.ncell))
    if self.thr_b is not None:
      return gauss_threshold(self.thr_a, self.thr_b, self.z)
    return np.asarray(self.thr_a, F32).reshape(self.nq, self.ncell).astype(F64)

  def oracle(self, skipna: bool) -> np.ndarray:
    """[nq][ncell][4] float64 point-wise scores from the oracle."""
    thr = self.thresholds()
    t = self.t.astype(F64)
    out = np.zeros((max(self.nq, 1), self.ncell, 4))
    with np.errstate(all='ignore'):
      if self.kind == 'ens':
        xs = self.members.astype(F64)
        for k in range(self.nq):
          out[k, :, 0] = orc.ens_brier_pointwise(xs, t, thr[k], 0, False, skipna)
          out[k, :, 1] = orc.ens_brier_pointwise(xs, t, thr[k], 0, True, skipna)
          out[k, :, 2] = orc.ens_ignorance_pointwise(xs, t, thr[k], 0, skipna)
          out[k, :, 3] = orc.ens_rps_part_pointwise(xs, t, thr[k], 0, skipna)
        return out
      f, s = self.mean.astype(F64), self.std.astype(F64)
      if self.nq == 0:
        out[0, :, 0] = orc.gaussian_crps_pointwise(f, s, t)
        out[0, :, 1] = s * s
        return out
      for k in range(self.nq):
        out[k, :, 0] = orc.gaussian_brier_pointwise(f, s, t, thr[k])
        out[k, :, 2] = orc.gaussian_ignorance_pointwise(f, s, t, thr[k])
        out[k, :, 3] = orc.gaussian_rps_part_pointwise(f, s, t, thr[k])
    return out

  def counts(self) -> tuple[np.ndarray, np.ndarray]:
    """Exact #{x > thr}, #{x < thr} per (threshold, cell) (float64 compares
    of float32 members are exact)."""
    thr = self.thresholds()
    xs = self.members.astype(F64)[None]
    with np.errstate(invalid='ignore'):
      return ((xs > thr[:, None]).sum(1), (xs < thr[:, None]).sum(1))


def _ens(name, members, t, *, thr_a, thr_b=None, z=None, nq=None,
         interleaved=False):
  members = np.asarray(members, F32)
  return Case(name, 'ens', np.asarray(t, F32),
              int(nq if nq is not None else np.size(z) if z is not None
                  else np.shape(thr_a)[0]),
              np.asarray(thr_a, F32), None if thr_b is None
              else np.asarray(thr_b, F32),
              None if z is None else np.asarray(z, F64), members=members,
              interleaved=interleaved)


def _near(lo, hi):
  """Candidate values around one bracket: below lo, lo, hi, above hi."""
  return [down(lo), F32(lo), F32(hi), up(hi)]


def fma_sensitive_cells(rs, n):
  """(mean, std, z, x) with mean + z * std == x (a float32) after two float64
  roundings, while the single rounding of fma(z, std, mean) is not x."""
  found = []
  while len(found) < n:
    x = F32(rs.uniform(1, 2) * 2.0 ** rs.randint(-4, 8))
    mean = F32(-x * rs.uniform(0.3, 0.7))
    std = F32(rs.uniform(0.2, 3))
    p = float(x) - float(mean)  # exact: both float32, similar exponents
    z0 = p / float(std)
    for dz in range(-4, 5):
      z = float(np.nextafter(z0, np.inf) if dz > 0 else z0)
      for _ in range(abs(dz)):
        z = float(np.nextafter(z, np.inf if dz > 0 else -np.inf))
      two = float(F64(mean) + F64(z) * F64(std))
      if two == float(x) and fma_single_rounding(mean, std, z) != float(x):
        found.append((mean, std, z, x))
        break
  return found


def bracket_cases(seed=0):
  """M = 8 (every probability and square is exact in float32), Gaussian-
  quantile thresholds, members and truth at and next to the bracket."""
  rs = np.random.RandomState(seed)
  m8 = 8
  z = np.array([stats.norm.ppf(0.3), 0.0, stats.norm.ppf(0.9),
                stats.norm.ppf(0.77)])
  n = 512
  mean = (rs.normal(size=n) * 10.0 ** rs.randint(-3, 4, size=n)).astype(F32)
  std = (rs.uniform(0.05, 4, size=n) * 10.0 ** rs.randint(-2, 3, size=n)
         ).astype(F32)
  std[::37] = 0  # thr = mean for every z
  # thresholds beyond float32 range: lo = FLT_MAX, hi = inf (and mirrored)
  mean[-4:] = [3e38, -3e38, 3e38, -3e38]
  std[-4:] = [1e38, 1e38, 3e38, 3e38]
  thr = gauss_threshold(mean, std, z)
  lo, hi = bracket(thr)
  members = np.empty((m8, n), F32)
  t = np.empty(n, F32)
  for c in range(n):
    k = c % z.size  # members placed around this cell's threshold k
    cand = _near(lo[k, c], hi[k, c])
    if lo[k, c] == hi[k, c]:
      cand.append(F32(lo[k, c]))  # thr itself, a float32 number
    if not np.isfinite(thr[k, c]) or abs(thr[k, c]) > FLT_MAX:
      cand += [F32(FLT_MAX), F32(-FLT_MAX), F32(np.inf), F32(-np.inf)]
    cand = np.array(cand, F32)
    members[:, c] = cand[rs.randint(0, cand.size, m8)]
    t[c] = cand[rs.randint(0, cand.size)]
  # fma-sensitive cells: members and truth at x
  fma = fma_sensitive_cells(rs, 16)
  fm = np.array([f[0] for f in fma], F32)
  fs = np.array([f[1] for f in fma], F32)
  fx = np.array([f[3] for f in fma], F32)
  fz = np.array([f[2] for f in fma])
  cases = [_ens('bracket_m8', members, t, thr_a=mean, thr_b=std, z=z)]
  # every fma cell c gets all 16 z; threshold k = c is its fma-sensitive one,
  # and its members and truth sit at (and next to) that threshold's x
  # (five members at x, two below, one above, and the truth off x: a
  # symmetric placement would give the same scores for either rounding)
  mem = np.stack([fx, down(fx), up(fx), fx, fx, down(fx), fx, fx])
  ft = np.where(np.arange(fx.size) % 2 == 0, up(fx), down(fx))
  cases.append(_ens('fma_m8', mem, ft, thr_a=fm, thr_b=fs, z=fz))
  return cases


def fma_cells_in(case) -> int:
  """Cells of `case` whose threshold k = cell index is a float32 number after
  two roundings but not after one (fma)."""
  n = 0
  for c in range(case.ncell):
    if c >= case.nq:
      break
    mean, std, z = case.thr_a[c], case.thr_b[c], case.z[c]
    two = float(F64(mean) + F64(z) * F64(std))
    if float(F32(two)) == two and fma_single_rounding(mean, std, z) != two:
      n += 1
  return n


def warp_cases(seed=1, nq=4):
  """Maps-kernel warps of three kinds, 32 cells each, M = 8:
  'strict'  every lane's thresholds lie strictly between two float32 values
            (the one-comparison shortcut);
  'onelane' the same cells with lane 5's std set to 0 (thr = its mean, a
            float32 number: the two-comparison path for the whole warp);
  'lastpass' strict for the first pass of 4 thresholds, but threshold 4
            (z = 0: thr = mean) is a float32 number, so only the pass of
            threshold 4 takes the two-comparison path.
  Returns (case, kinds) with kinds[w] the kind of warp w."""
  rs = np.random.RandomState(seed)
  z = np.array([stats.norm.ppf(q) for q in (0.1, 0.35, 0.6, 0.85)][:nq] +
               [0.0])
  nwarp = 12
  n = 32 * nwarp
  kinds = ['strict', 'onelane', 'lastpass'] * (nwarp // 3)
  base_mean = rs.normal(scale=5, size=32).astype(F32)
  base_std = rs.uniform(0.5, 2, size=32).astype(F32)
  mean = np.tile(base_mean, nwarp)
  std = np.tile(base_std, nwarp)
  for w, kind in enumerate(kinds):
    if kind == 'onelane':
      std[32 * w + 5] = 0
  thr = gauss_threshold(mean, std, z)
  lo, hi = bracket(thr)
  # make the strict lanes really strict for thresholds 0..3 (redraw is not
  # needed in practice; assert it below)
  members = np.empty((8, n), F32)
  t = np.empty(n, F32)
  rs2 = np.random.RandomState(seed + 100)
  cells_a = []
  for c in range(32):
    k = c % 4
    cand = np.array(_near(lo[k, c], hi[k, c]), F32)
    cells_a.append((cand[rs2.randint(0, 4, 8)], cand[rs2.randint(0, 4)]))
  for w in range(nwarp):
    for c in range(32):
      members[:, 32 * w + c], t[32 * w + c] = cells_a[c]
  case = _ens('warps', members, t, thr_a=mean, thr_b=std, z=z)
  return case, kinds


def warp_strictness(case):
  """Per warp of the maps kernel and per pass of 4 / 2 / 1 thresholds: True
  if every lane's thresholds of that pass are strict (lo < hi)."""
  lo, hi = bracket(case.thresholds())
  strict = lo < hi  # [nq][ncell]
  res = []
  q0 = 0
  while q0 < case.nq:
    tq = 4 if case.nq - q0 >= 4 else 2 if case.nq - q0 >= 2 else 1
    s = strict[q0:q0 + tq].all(0).reshape(-1, 32).all(1)
    res.append(s)
    q0 += tq
  return res


def field_cases(seed=2):
  """Field thresholds (thr_b == NULL): integer-valued members, truth and
  thresholds, so ties x == thr are common; NaN thresholds."""
  rs = np.random.RandomState(seed)
  n, m = 300, 6
  members = rs.randint(-3, 4, size=(m, n)).astype(F32)
  t = rs.randint(-3, 4, size=n).astype(F32)
  thr = rs.randint(-3, 4, size=(3, n)).astype(F32)
  thr[rs.rand(3, n) < 0.1] = np.nan
  t[::29] = np.nan
  return [_ens('field_int', members, t, thr_a=thr)]


def member_count_cases(seed=3):
  """M in {1, 2, 24, 25, 26, 49, 51, 64, 65, 257, 5000}, both layouts, cells
  with nvalid = 0, 1 and M, NaN truth, +-Inf members and truth."""
  rs = np.random.RandomState(seed)
  cases = []
  for m in (1, 2, 24, 25, 26, 49, 51, 64, 65, 257, 5000):
    n = 64 if m < 1000 else 16
    members = rs.normal(size=(m, n)).astype(F32)
    t = rs.normal(size=n).astype(F32)
    nan = rs.rand(m, n) < 0.2
    nan[:, 0] = True                 # nvalid = 0
    nan[:, 1] = True
    nan[rs.randint(m), 1] = False    # nvalid = 1
    nan[:, 2:6] = False              # nvalid = M
    members[nan] = np.nan
    members[0, 6] = np.inf
    members[-1, 7] = -np.inf
    t[8], t[9], t[10] = np.nan, np.inf, -np.inf
    # thresholds: field form with a few exact hits on members
    thr = rs.normal(size=(2, n)).astype(F32)
    thr[0, 11:14] = members[0, 11:14]
    for inter in (False, True):
      cases.append(_ens(f'M{m}_{"interleaved" if inter else "member_major"}',
                        members, t, thr_a=thr, interleaved=inter))
  return cases


def threshold_count_cases(seed=4):
  """nq in {1, 2, 3, 4, 5, 7, 9}: every mix of passes of 4 / 2 / 1."""
  rs = np.random.RandomState(seed)
  n, m = 96, 10
  members = rs.normal(size=(m, n)).astype(F32)
  t = rs.normal(size=n).astype(F32)
  mean = rs.normal(size=n).astype(F32)
  std = rs.uniform(0.5, 1.5, size=n).astype(F32)
  cases = []
  for nq in (1, 2, 3, 4, 5, 7, 9):
    z = stats.norm.ppf(np.linspace(0.05, 0.95, nq))
    cases.append(_ens(f'nq{nq}_gauss', members, t, thr_a=mean, thr_b=std,
                      z=z))
    thr = rs.normal(size=(nq, n)).astype(F32)
    cases.append(_ens(f'nq{nq}_field', members, t, thr_a=thr))
  return cases


# -- Gaussian ------------------------------------------------------------------
def z_for_tail(tail):
  """z > 0 with 0.5 erfc(z / sqrt 2) = tail (float64)."""
  return float(-stats.norm.ppf(tail))


def gaussian_z_grid():
  """Standard-normal offsets of the threshold from the forecast mean."""
  zs = [0.0, 1e-30, 0.5, 1.0, 3.0, 6.0, 8.0, 20.0, 40.0, np.inf]
  zs += list(np.linspace(5.15, 5.25, 11))            # the 1e-7 switch
  zs += [z_for_tail(SATURATION * f) for f in
         (0.5, 0.9, 0.99, 0.999, 1.001, 1.01, 1.1, 2.0)]  # 1 - cdf saturation
  zs += [10.0, 13.0, 14.0, 16.0, 30.0, 37.0, 37.6, 37.75]
  zs = np.array(zs)
  return np.concatenate([zs, -zs[zs != 0]])


def gaussian_cases(seed=5):
  """Forecast N(mean, std) against Gaussian-quantile and field thresholds.
  Cells are built from a standard offset zt: thr - mean = zt * std, with the
  truth on each side of the threshold or NaN."""
  rs = np.random.RandomState(seed)
  zt = gaussian_z_grid()
  sides = (-1, 1, np.nan)
  rows = [(z, s) for z in zt for s in sides]
  n = len(rows)
  cmean = (rs.normal(size=n) * 3).astype(F32)      # climatological mean
  cstd = rs.uniform(0.5, 2, size=n).astype(F32)    # climatological std
  zq = np.array([stats.norm.ppf(0.8)])
  thr = gauss_threshold(cmean, cstd, zq)[0]
  std = rs.uniform(0.3, 2, size=n).astype(F32)
  zcol = np.array([r[0] for r in rows])
  # |z| < 1e-6: thr = 0 exactly, so the float32 mean keeps z
  small = np.abs(zcol) < 1e-6
  cmean[small], cstd[small] = 0, 0
  thr = gauss_threshold(cmean, cstd, zq)[0]
  with np.errstate(invalid='ignore', over='ignore'):
    mean = (thr - zcol * std.astype(F64)).astype(F32)
  side = np.array([r[1] for r in rows])
  lo, hi = bracket(thr)
  t = np.where(side > 0, up(hi), np.where(side < 0, down(lo), np.nan)).astype(
      F32)
  # the special values
  extra_std = np.array([0, 1e-30, 1e-3, 1, 1e3, np.inf, np.nan], F32)
  k = extra_std.size
  e_cm = np.zeros(3 * k + 6, F32)
  e_cs = np.ones(3 * k + 6, F32)
  e_mean = np.concatenate([np.full(k, -0.5), np.full(k, 0.0), np.full(k, 2.0),
                           [np.nan, np.inf, -np.inf, 0.0, 0.0, 0.0]]).astype(F32)
  e_std = np.concatenate([extra_std] * 3 + [np.ones(6)]).astype(F32)
  e_t = rs.normal(size=3 * k + 6).astype(F32)
  e_cm[-3] = np.nan                   # NaN threshold (NaN climatology cell)
  e_cs[-2] = np.nan
  e_cm[-1] = 3e38                     # threshold beyond float32 range
  e_cs[-1] = 3e38
  cm = np.concatenate([cmean, e_cm])
  cs = np.concatenate([cstd, e_cs])
  gmean = np.concatenate([mean, e_mean])
  gstd = np.concatenate([std, e_std])
  gt = np.concatenate([t, e_t])
  cases = [Case('gauss_quantile', 'gauss', gt, 1, cm, cs, zq, mean=gmean,
                std=gstd)]
  with np.errstate(over='ignore'):
    field = gauss_threshold(cm, cs, zq)[0].astype(F32)[None]
  cases.append(Case('gauss_field', 'gauss', gt, 1, field, mean=gmean,
                    std=gstd))
  cases.append(Case('gauss_crps', 'gauss', gt, 0, None, mean=gmean, std=gstd))
  # several thresholds, with a pass mix of 4 + 2 + 1
  z7 = stats.norm.ppf(np.linspace(0.02, 0.98, 7))
  cases.append(Case('gauss_quantile_nq7', 'gauss', gt, 7, cm, cs, z7,
                    mean=gmean, std=gstd))
  return cases


# ---------------------------------------------------------------------------
# The kernel's float32 z and the error bounds
# ---------------------------------------------------------------------------
ULP_ERFCF, ULP_LOGF, ULP_LOG1PF, ULP_EXPF = 4, 1, 1, 2  # CUDA math API, float32
ULP_ERFC64 = 5                                         # double erfc
C_SQRT1_2 = float(F32(0.70710678))  # the kernel's float32 1 / sqrt(2)
D_C = abs(C_SQRT1_2 * np.sqrt(2.0) - 1.0)  # its relative error (2.5e-8)


def emulate_z(thr, mean, std):
  """The kernel's zn = float32(thr - double(mean)) * (1.f / std)."""
  with np.errstate(all='ignore'):
    d = (np.asarray(thr, F64) - np.asarray(mean, F32).astype(F64)).astype(F32)
    rsd = F32(1) / np.asarray(std, F32)
    return d * rsd


def emulate_tail(zn):
  """(a, tail): a = |zn| * 0.70710678f in float32, tail = erfc(a) / 2 in
  float64 (the float32 path's argument, evaluated exactly)."""
  with np.errstate(all='ignore'):
    a = (np.abs(zn) * F32(C_SQRT1_2)).astype(F32)
  return a, 0.5 * special.erfc(a.astype(F64))


def reference_scores(tail, upside, t_gt, t_lt):
  """The reference's formulas (metrics.py:963-1118) in float64, given
  tail = min(cdf, 1 - cdf) and which side cdf is on."""
  with np.errstate(all='ignore'):
    cdf = np.where(upside, 1.0 - tail, tail)
    pe = 1.0 - cdf
    brier = (pe - t_gt) ** 2
    rps = (cdf - t_lt) ** 2
    ign = -np.log(np.where(t_gt, pe, cdf))
  return brier, ign, rps


def score_bounds(tail, rel_tail, upside, t_gt, t_lt, brier, ign, rps):
  """Absolute bounds on |kernel - reference| given the relative error of the
  tail the kernel works from (`rel_tail`).  Each score is a function of either
  p = tail (relative error rel_tail) or p = 1 - tail, which the float32 path
  rounds once (absolute u); the square and the final float32 rounding add
  2u relative; logf / log1pf add one ulp (2u relative) of the result; 2^-149
  covers results in the float32 subnormal range."""
  tiny = 2.0 ** -149
  dtail = rel_tail * tail + 2.0 ** -52  # + the float64 1 - (1 - tail) step
  one_m_b = t_gt == upside                # brier's |db| is 1 - tail
  one_m_r = t_lt != upside                # rps's |dr| is 1 - tail
  with np.errstate(all='ignore'):
    db = np.sqrt(brier)
    dr = np.sqrt(rps)
    e_b = np.where(one_m_b, dtail + U, dtail)
    e_r = np.where(one_m_r, dtail + U, dtail)
    bb = 2 * db * e_b + e_b ** 2 + 2 * U * brier + tiny
    br = 2 * dr * e_r + e_r ** 2 + 2 * U * rps + tiny
    # ignorance: -log(tail) moves by rel_tail; -log(1 - tail) by
    # dtail / (1 - tail) <= 2 dtail
    tail_side = t_gt == upside
    bi = np.where(tail_side, rel_tail + 2.0 ** -52 / np.maximum(tail, 1e-300),
                  2 * dtail) + 2 * U * ign + tiny
  return bb, bi, br


def rel_tail_from_a(a, rel_a):
  """|d ln erfc(a)| for a relative error rel_a of a:
  |d ln erfc / da| = (2 / sqrt pi) e^{-a^2} / erfc(a) <= a + sqrt(a^2 + 2)
  (the Mills-ratio bound), so the relative tail error is at most
  (a + sqrt(a^2 + 2)) * a * rel_a."""
  a = np.abs(np.asarray(a, F64))
  return (a + np.sqrt(a * a + 2)) * a * rel_a


def reduction_case(seed=6, nfield=3, m=10):
  """Fields of 13 rows (not a multiple of the 4- or 8-row block) of 150
  columns (row segments longer than 64 cells whose lengths are not multiples
  of 32) in rows of stride 160; three regions over three longitude boxes,
  column and cell weights with zeros, and NaN in every zero-weight cell.
  Returns a dict of float32 arrays and the WeightSpec arguments (cell_w is a
  host array: the caller passes its device or host address)."""
  rs = np.random.RandomState(seed)
  nrow, ncol, stride = 13, 150, 160
  cells = nrow * stride
  col_w = rs.uniform(0.5, 1.5, ncol).astype(F32)
  col_w[[3, 77]] = 0
  cell_w = rs.uniform(0.5, 1.5, (nrow, ncol)).astype(F32)
  cell_w[rs.rand(nrow, ncol) < 0.05] = 0
  row_w = rs.uniform(0.2, 1, (3, nrow))
  row_w[1, 4] = 0
  seg = [0, 37, 120, 150]  # segment lengths 37, 83, 30
  seg_w = np.array([[1, 0, 1], [0.5, 1, 0.25], [1, 1, 1]], F64)
  zero = (col_w[None] * cell_w == 0)
  def field(*shape, scale=1.0):
    a = (rs.normal(size=shape + (nrow, stride)) * scale).astype(F32)
    a[..., :ncol][..., zero] = np.nan
    return a
  x = field(m, nfield)
  t = field(nfield)
  x[rs.rand(*x.shape) < 0.02] = np.nan  # a few NaN members in weighted cells
  mean, std = field(nfield), np.abs(field(nfield)) + F32(0.3)
  cm, cs = field(nfield), np.abs(field(nfield)) + F32(0.5)
  thr = field(4, nfield)
  return dict(nrow=nrow, ncol=ncol, stride=stride, cells=cells, x=x, t=t,
              mean=mean, std=std, cm=cm, cs=cs, thr=thr, m=m, nfield=nfield,
              weights=dict(nrow=nrow, ncol=ncol, row_w=row_w, seg_start=seg,
                           seg_w=seg_w, col_w=col_w, row_stride=stride),
              cell_w=cell_w)


def ens_emulate(case, skipna):
  """The kernel's Brier and RPS part in float32 with IEEE quotients (the
  Newton-step quotient equals them for counts up to 1551): [nq][ncell] x 2,
  and the counts (#{x > lo}, #{x < hi}, nvalid) it forms."""
  lo, hi = bracket(case.thresholds())
  xs = case.members[None]
  with np.errstate(all='ignore'):
    c_gt = (xs > lo[:, None]).sum(1).astype(F32)
    c_lt = (xs < hi[:, None]).sum(1).astype(F32)
    nvalid = (~np.isnan(case.members)).sum(0).astype(F32)
    m = F32(case.nmember)
    nv = nvalid if skipna else m
    pf = c_gt / nv
    if not skipna:
      pf = np.where(nvalid < m, F32(np.nan), pf)
    t = case.t[None]
    tp = np.where(np.isnan(t), F32(np.nan), (t > lo).astype(F32))
    d = (pf - tp).astype(F32)
    dr = (c_lt / m - (t < hi).astype(F32)).astype(F32)
    return (d * d).astype(F32), (dr * dr).astype(F32), (c_gt, c_lt, nvalid)


def geometry_1x1():
  return _lib.WeightSpec(1, 1, np.ones((1, 1)), [0, 1], np.ones((1, 1)))

"""Seeded single-point cases for the ensemble point statistics of K2
(csrc/ens_metrics.cu, csrc/ens_point.cuh), K6e (csrc/ens_maps.cu) and K2b
(csrc/ens_big.cu), with float64 references and per-statistic error bounds
derived from the kernels' operation order.  Importable without a GPU.

A case is one member count M: `x` [M][n] float32 members of n grid points,
`t` [n] float32 truth, and a label per point.  Points come in adjacent pairs
with the same label, so a 1 x 2 geometry (ens_pair_kernel's two points per
lane) averages two points of one family.

Families (labels):
  mag:<mean>:<ratio>:<in|out>  members of mean 0, 280, 5e4, 1e5 or -5e4 and
      spread ratio * |mean| (1 for mean 0), ratio from 1e-4 to 1; truth drawn
      like a member (in) or 100 spreads away (out)
  equal        all members equal (spread and variance exactly 0)
  pm0          members +0 and -0 (every statistic exactly 0 against t = 0)
  two          M = 2: spread |x1 - x2|
  ties         members from three values
  outlier      one member 1e6 spreads from the others
  nan1 / nanall_but1 / nanall / nant    one NaN member, all but one NaN, all
      NaN, NaN truth
  pinf / ninf / tpinf / tninf    one +inf or -inf member, +inf or -inf truth
Finite values stay at or below 1e30.

The reference follows the oracle (oracle/wb2_oracle.py): the spread is the
rank form 2 mean((2 r - M - 1) x) / (M - 1) with oracle.rankdata's ordinal
ranks, in float64 on the float32-rounded inputs, and under skipna divides by
the valid count while the coefficients keep the full M (metrics.py's
_get_n_ensemble).

Bounds (u = 2^-24; D = max_m |x_m - xbar| the point's dispersion; delta the
float32 mean's error, at most (n + 1) u mean|x_m| over the n valid members;
every kernel path sums the members serially (K2b: per lane, then a butterfly,
fewer levels than members) and scales by 1 / M as a float32 reciprocal or an
IEEE division):
  skill    (M + 4) u skill: M roundings of the terms and the serial sum, two of
           the scaling.
  spread   the rank sum is formed on y_m = fl(x_m - mean); its FMA chain's
           partial sums are bounded by A = sum_i |c_i| (|y_(i)| + delta), so
           (M + 4) u 2 A / (M (M - 1)) + 3 u |spread|.  A is proportional to
           the dispersion, not to |x|.  The (a + b) - lo networks (twin, pair)
           add 4 u (D + delta) per comparator level a value passes through,
           times M / (M - 1).  Under skipna with n < M valid members the shift
           term mean n (n - M) does not cancel: + (n + 4) u mean|x_m|
           2 |n - M| / (M - 1).
  mse      with d' = delta + u (|t - xbar| + delta): 2 |t - xbar| d' + d'^2
           + 3 u (t - xbar)^2.
  var      n delta^2 / (n - 1) + (n + 5) u (var + n delta^2 / (n - 1)).
  deb      bound(mse) + bound(var) / M + 2 u |deb| + u var / M.
The same bounds are stated in DESIGN.md (K2, section 5)."""
from __future__ import annotations

import dataclasses
import warnings

import numpy as np

from region_cases import PAIR_MP, U

STATS = ('skill', 'spread', 'mse', 'var', 'deb')
MEMBER_COUNTS = (1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 16, 17, 20, 21, 32, 33, 49,
                 50, 51, 63, 64, 65, 100, 1000, 1551)
MEANS = (0.0, 280.0, 5e4, 1e5, -5e4)
RATIOS = (1e-4, 1e-3, 1e-2, 1e-1, 1.0)
# all-equal values: powers of two, so the float32 sum of M copies is exact and
# so is the kernels' mean (scaled by the float32 reciprocal of M on the paths
# without skipna, which rounds back to c only for some c and M: 5e4 at M = 7
# comes out one ulp off, and its variance is then not exactly 0)
EQUAL_VALUES = (0.5, 256.0, 65536.0, -65536.0, 131072.0, -1.0)


@dataclasses.dataclass
class PointCase:
  M: int
  x: np.ndarray        # [M][n] float32
  t: np.ndarray        # [n] float32
  labels: list         # [n]

  @property
  def n(self):
    return self.t.size

  def mask(self, prefix):
    return np.array([l.split(':')[0] == prefix for l in self.labels])

  def finite(self):
    return np.isfinite(self.x).all(axis=0) & np.isfinite(self.t)


def _pair(xs, ts, labels, x, t, label):
  """Appends two points of one family (x: [M][2], t: [2])."""
  xs.append(np.asarray(x, np.float64))
  ts.append(np.asarray(t, np.float64))
  labels += [label, label]


def point_case(M: int) -> PointCase:
  rs = np.random.RandomState(1000 + M)
  xs, ts, labels = [], [], []
  for mu in MEANS:
    for ratio in RATIOS:
      s = ratio * abs(mu) if mu else 1.0
      for where in ('in', 'out'):
        x = mu + s * rs.standard_normal((M, 2))
        t = (mu + s * rs.standard_normal(2) if where == 'in' else
             mu + 100 * s * np.where(rs.rand(2) < 0.5, -1.0, 1.0))
        _pair(xs, ts, labels, x, t, f'mag:{mu:g}:{ratio:g}:{where}')
  for c in EQUAL_VALUES:
    _pair(xs, ts, labels, np.full((M, 2), c), [c + 1.0, c - 2.0], 'equal')
  pm = np.where(np.arange(M)[:, None] % 2 == 0, 0.0, -0.0) * np.ones((M, 2))
  _pair(xs, ts, labels, pm, [0.0, -0.0], 'pm0')
  if M == 2:
    _pair(xs, ts, labels, 280 + rs.standard_normal((2, 2)), [280.0, 281.0],
          'two')
  vals = np.array([5e4 - 5, 5e4, 5e4 + 2.5])
  _pair(xs, ts, labels, vals[rs.randint(3, size=(M, 2))], [5e4, 5e4 + 1],
        'ties')
  x = 280 + rs.standard_normal((M, 2))
  x[rs.randint(M), 0] = 280 + 1e6
  x[rs.randint(M), 1] = 280 - 1e6
  _pair(xs, ts, labels, x, [280.5, 279.5], 'outlier')

  def base():
    return 5e4 + 5 * rs.standard_normal((M, 2)), 5e4 + 5 * rs.standard_normal(2)

  x, t = base()
  x[rs.randint(M), :] = np.nan
  _pair(xs, ts, labels, x, t, 'nan1')
  if M > 1:
    x, t = base()
    keep = rs.randint(M)
    x[np.arange(M) != keep, :] = np.nan
    _pair(xs, ts, labels, x, t, 'nanall_but1')
  x, t = base()
  _pair(xs, ts, labels, np.full((M, 2), np.nan), t, 'nanall')
  x, t = base()
  _pair(xs, ts, labels, x, [np.nan, np.nan], 'nant')
  for lab, v in (('pinf', np.inf), ('ninf', -np.inf)):
    x, t = base()
    x[rs.randint(M), :] = v
    _pair(xs, ts, labels, x, t, lab)
  for lab, v in (('tpinf', np.inf), ('tninf', -np.inf)):
    x, t = base()
    _pair(xs, ts, labels, x, [v, v], lab)
  x = np.concatenate(xs, axis=1).astype(np.float32)
  t = np.concatenate(ts).astype(np.float32)
  assert np.nanmax(np.abs(np.where(np.isinf(x), 0, x))) <= 1e30
  return PointCase(M, x, t, labels)


def cases():
  return {M: point_case(M) for M in MEMBER_COUNTS}


# ---- dispatch ----------------------------------------------------------------------
def bucket(M):
  """(MP, exact) of launch_ens / launch_ens_maps, or (None, False) for K2b."""
  if M > 64:
    return None, False
  mp = next(b for b in PAIR_MP if M <= b)
  return mp, M == mp


def metrics_path(M, skipna, env=None, layout='pair'):
  """Path of wb2_ens_metrics for one of the GPU test's layouts: 'pair' (1 x 2
  geometry, even offsets and member stride: ens_pair_kernel eligible) or
  'odd' (odd offsets).  Restates region_cases._ens_plan on a Case of that
  shape, so the dispatch rules live in one place."""
  import region_cases as rc  # pylint: disable=import-outside-toplevel
  n = 2
  shift = 1 if layout == 'odd' else 0
  case = rc.Case('point', 'ens', 1, n, n, np.ones((1, 1)),
                 np.array([0, n], np.int32), np.ones((1, 1)), skipna=skipna,
                 nmember=M, member_stride=2 * 64)
  case.offsets = {'x': np.array([shift]), 't': np.array([shift])}
  return rc.plan(case, env or {}).path


def maps_path(M, skipna):
  """ens_maps_kernel's network: 'twin' when kTwinSortOk, else 'scalar'."""
  mp, exact = bucket(M)
  return 'twin' if (exact and not skipna and mp >= 8 and mp % 2 == 0) else 'scalar'


NETWORK_PATHS = ('twin', 'pair')   # (a + b) - lo comparators


# ---- float64 reference -------------------------------------------------------------
def reference(case: PointCase, skipna: bool):
  """name -> [n] float64 point statistics, the oracle's formulas restated in
  float64 (spread on oracle.rankdata)."""
  from oracle import wb2_oracle as orc  # pylint: disable=import-outside-toplevel
  x = case.x.astype(np.float64)
  t = case.t.astype(np.float64)
  M = case.M
  with warnings.catch_warnings(), np.errstate(invalid='ignore', divide='ignore'):
    warnings.simplefilter('ignore', RuntimeWarning)
    mean = np.nanmean if skipna else np.mean
    skill = mean(np.abs(t[None] - x), axis=0)
    if M < 2:
      spread = np.zeros(case.n)
    else:
      rank = orc.rankdata(x, 0)
      spread = 2 * mean((2 * rank - M - 1) * x, axis=0) / (M - 1)
    xbar = mean(x, axis=0)
    mse = (t - xbar) ** 2
    var = ((np.nanvar if skipna else np.var)(x, axis=0, ddof=1) if M > 1
           else np.full(case.n, np.nan))
    deb = mse - var / M
  return dict(skill=skill, spread=spread, mse=mse, var=var, deb=deb)


def brute_force_spread(case: PointCase):
  """mean_ij |x_i - x_j| M / (M - 1) (metrics_test.py's brute force), float64."""
  x = case.x.astype(np.float64)
  M = case.M
  if M < 2:
    return np.zeros(case.n)
  with np.errstate(invalid='ignore'):
    d = np.abs(x[:, None] - x[None])
  return d.mean(axis=(0, 1)) * M / (M - 1)


# ---- bounds ------------------------------------------------------------------------
def _depth(comparators, n):
  """Comparator levels of a network: the longest chain through any position."""
  lvl = np.zeros(n, int)
  for a, b in comparators:
    lvl[a] = lvl[b] = max(lvl[a], lvl[b]) + 1
  return int(lvl.max()) if n else 0


def network_depth(mp):
  import re  # pylint: disable=import-outside-toplevel
  import os  # pylint: disable=import-outside-toplevel
  inc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                     'weatherbench2_b200', 'csrc', 'sort_networks.inc')
  body = re.search(rf'struct SortNet<{mp}> \{{(.*?)\n\}};', open(inc).read(),
                   re.S).group(1)
  comps = [(int(a), int(b)) for a, b in re.findall(r'CE\((\d+),(\d+)\)', body)]
  return _depth(comps, mp)


def bounds(case: PointCase, skipna: bool, path: str, ref=None):
  """name -> [n] float64 bound on |kernel - reference| at every point (NaN
  where the reference is not finite: those points are compared by pattern)."""
  ref = reference(case, skipna) if ref is None else ref
  x = case.x.astype(np.float64)
  t = case.t.astype(np.float64)
  M = case.M
  with warnings.catch_warnings(), np.errstate(invalid='ignore', divide='ignore'):
    warnings.simplefilter('ignore', RuntimeWarning)
    valid = ~np.isnan(x) if skipna else np.ones_like(x, bool)
    n = valid.sum(axis=0).astype(np.float64)
    xv = np.where(valid, x, 0.0)
    xbar = xv.sum(axis=0) / n
    absmean = np.abs(xv).sum(axis=0) / n
    delta = (n + 1) * U * absmean
    y = np.where(valid, np.abs(x - xbar), 0.0)
    D = y.max(axis=0)
    out = {}
    out['skill'] = (M + 4) * U * np.abs(ref['skill'])
    if M < 2:
      out['spread'] = np.zeros(case.n)
    else:
      ys = np.sort(np.where(valid, x - xbar, np.inf), axis=0)
      coef = np.abs(2 * np.arange(1, M + 1) - M - 1).astype(np.float64)[:, None]
      A = np.where(np.arange(M)[:, None] < n[None], coef * (np.abs(ys) + delta),
                   0.0).sum(axis=0)
      sp = (M + 4) * U * 2 * A / (n * (M - 1)) + 3 * U * np.abs(ref['spread'])
      if path in NETWORK_PATHS:
        mp, _ = bucket(M)
        sp = sp + network_depth(mp) * 4 * U * (D + delta) * M / (M - 1)
      if skipna:
        sp = sp + (n + 4) * U * absmean * 2 * np.abs(n - M) / (M - 1)
      out['spread'] = sp
    dm = np.abs(t - xbar)
    d1 = delta + U * (dm + delta)
    out['mse'] = 2 * dm * d1 + d1 ** 2 + 3 * U * dm ** 2
    shift = n * delta ** 2 / (n - 1)
    out['var'] = shift + (n + 5) * U * (np.abs(ref['var']) + shift)
    out['deb'] = (out['mse'] + out['var'] / M + 2 * U * np.abs(ref['deb']) +
                  U * np.abs(ref['var']) / M)
  return out


def exact_expectations(case: PointCase, skipna: bool):
  """name -> (mask [n], value): points where a statistic is exact."""
  eq = case.mask('equal') | case.mask('pm0')
  out = {'spread': (eq, 0.0)}
  if case.M > 1:
    out['var'] = (eq, 0.0)
  if case.M == 1:  # spread 0 whatever the member (metrics.py:788-789)
    out['spread'] = (np.ones(case.n, bool), 0.0)
  pm = case.mask('pm0')
  out['skill'] = (pm, 0.0)
  out['mse'] = (pm, 0.0)
  return out

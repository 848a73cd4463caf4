"""Seeded SEEPS cases (K9, csrc/seeps.cu), the reference they are held to, and
NumPy models of the kernel's arithmetic.

SEEPS is categorical: a comparison that goes the other way moves a cell from
one category to another and changes its score by O(1).  That only happens
within one rounding of a threshold, so the cases put values there on purpose.

Raw cases (`raw_cases`) are what `ctx.seeps_maps` takes: forecast and truth
fields [nfield][nrow][ncol], wet-threshold slabs [nwet][nrow][wet_stride] with
the slab of every field, the dry fraction p1 [nrow][ncol], ngroup and skipna.
Each case names the edges it claims (`EDGES`), and `reached_edges` finds them
in the arrays:
- realistic 24-hour precipitation in metres on 121 x 240 and a 0.25 degree
  band of 1440 longitudes from 2 S to 22 N: 40-60 % exact zeros, gamma-distributed wet amounts,
  tiny positive values and small negatives as packed reanalysis data has; wet
  thresholds of 0.5 to 20 mm; p1 on a latitude profile from below 0.1 (wet
  tropics) to above 0.85 (deserts); lead times of 1 to 10 days over init
  times in a leap year;
- float32 values one ulp below, at and one ulp above the dry and the wet
  threshold, +-0, negatives, NaN and +-inf, on the forecast and on the truth
  side, so every cell of the 3 x 3 table and "no category" occur;
- wet below, equal to, NaN, 0 and inf; p1 at float32(0.1) / float32(0.85) and
  their neighbours, 0, 1 and NaN;
- float64 precipitation strictly between the float32 neighbours of a
  threshold, float64 p1 strictly between the neighbours of float32(0.1) and
  float32(0.85), and five (forecast, truth, wet, p1) dtype mixes;
- ngroup 1 and > 1 with skipna both ways, an all-NaN series, a wet
  climatology with its own row stride and many outputs.

Lookup cases (`lookup_cases`) are datasets for the operators: valid times on
Feb 29, Dec 31 of leap and non-leap years and across the year boundary,
6-hourly data against hours 0/6/12/18, 24-hourly data against hour 0 only, an
unsorted and a subset `dayofyear`, and a valid hour the climatology lacks
(KeyError, as `.sel` raises).

The reference (`reference`) is `oracle.seeps_pointwise` on the operands in
their own dtypes followed by Metric.compute's time mean, rounded to float32.
`kernel_model` restates the kernel's arithmetic; `old_kernel_model` the kernel
before it read operands in their own dtypes (every operand cast to float32,
the scoring matrix in float64 from the float32 p1, each step rounded to
float32 before the time mean).
"""
from __future__ import annotations

import dataclasses
import warnings

import numpy as np
import pandas as pd

from oracle import wb2_oracle as orc

F32, F64 = np.dtype(np.float32), np.dtype(np.float64)
DRY_MM = 0.25
NAME = 'total_precipitation_24hr'
DAY = np.timedelta64(1, 'D').astype('timedelta64[ns]')
HOUR = np.timedelta64(1, 'h').astype('timedelta64[ns]')

VALUE_EDGES = ('below_dry', 'at_dry', 'above_dry', 'below_wet', 'at_wet',
               'above_wet', 'pos_zero', 'neg_zero', 'negative', 'nan',
               'pos_inf', 'neg_inf', 'no_category', 'f64_near_dry',
               'f64_near_wet')
CELL_EDGES = tuple(f'cell_{a}{b}' for a in 'dlh' for b in 'dlh')
EDGES = frozenset(
    [f'{s}_{e}' for s in 'ft' for e in VALUE_EDGES] + list(CELL_EDGES) + [
        'two_categories', 'wet_below_dry', 'wet_eq_dry', 'wet_nan',
        'wet_zero', 'wet_inf', 'p1_at_min', 'p1_below_min', 'p1_above_min',
        'p1_at_max', 'p1_below_max', 'p1_above_max', 'p1_zero', 'p1_one',
        'p1_nan', 'p1_masked_low', 'p1_masked_high', 'p1_f64_near_min',
        'p1_f64_near_max', 'precip32_at_rounded_wet64', 'exact_zero',
        'tiny_positive', 'small_negative', 'wet_0.5_to_20mm',
        'mix_32_32_32_32', 'mix_64_64_64_64', 'mix_64_32_32_32',
        'mix_32_32_64_32', 'mix_32_32_32_64', 'ngroup1_skipna0',
        'ngroup1_skipna1', 'ngroupN_skipna0', 'ngroupN_skipna1',
        'all_nan_series', 'wet_row_stride', 'many_outputs', 'partial_block'])


@dataclasses.dataclass
class Case:
  name: str
  edges: frozenset
  f: np.ndarray        # [nfield][nrow][ncol]
  t: np.ndarray
  wet: np.ndarray      # [nwet][nrow][wet_stride]
  p1: np.ndarray       # [nrow][ncol]
  wf: np.ndarray       # [nfield] wet slab at the forecast's valid time
  wt: np.ndarray       # ... at the truth's
  ngroup: int = 1
  skipna: bool = False
  dry_mm: float = DRY_MM
  min_p1: float = 0.1
  max_p1: float = 0.85

  @property
  def nfield(self):
    return self.f.shape[0]

  @property
  def nout(self):
    return self.nfield // self.ngroup

  @property
  def nrow(self):
    return self.f.shape[1]

  @property
  def ncol(self):
    return self.f.shape[2]

  @property
  def dry(self):
    """The dry threshold in metres, as SpatialSEEPS passes it."""
    return self.dry_mm / 1000.0

  def wet_at(self, which):
    """The wet threshold of every field, [nfield][nrow][ncol]."""
    return self.wet[:, :, :self.ncol][self.wf if which == 'f' else self.wt]


def _quiet():
  ctx = warnings.catch_warnings()
  ctx.__enter__()
  warnings.simplefilter('ignore', RuntimeWarning)
  return ctx


# ---- reference and models --------------------------------------------------------
def point_reference(case):
  """float64 [nfield][nrow][ncol]: SpatialSEEPS.compute_chunk per field."""
  ctx = _quiet()
  try:
    with np.errstate(all='ignore'):
      return orc.seeps_pointwise(case.f, case.t, case.wet_at('f'),
                                 case.wet_at('t'), case.p1, case.dry_mm,
                                 case.min_p1, case.max_p1)
  finally:
    ctx.__exit__(None, None, None)


def reference(case):
  """float32 [nout][nrow][ncol]: the reference's maps averaged over each group
  of ngroup fields (Metric.compute), rounded to float32."""
  pt = point_reference(case).reshape((case.nout, case.ngroup) + case.f.shape[1:])
  dims = ('out', 'group', 'row', 'col')
  ctx = _quiet()
  try:
    r, _ = orc.time_mean(pt, dims, skipna=case.skipna, avg_dim='group')
  finally:
    ctx.__exit__(None, None, None)
  return r.astype(np.float32)


def categories(x, dry, wet):
  """(dry, light, heavy, nan) of `x` against the Python-float `dry` and the
  array `wet`, compared in double after widening: the promoted comparison,
  with `dry` rounded to x's dtype first."""
  d = np.float64(x.dtype.type(dry))
  xd, wd = x.astype(np.float64), np.asarray(wet).astype(np.float64)
  return xd < d, (xd > d) & (xd < wd), xd >= wd, np.isnan(xd)


def scoring_matrix(p1):
  """0.5 * the scoring matrix in p1's dtype, each operation rounded in it
  (metrics.py:487-499), widened to float64: [3][3][nrow][ncol]."""
  P = p1.dtype.type
  with np.errstate(all='ignore'):
    h, one = P(0.5), P(1)
    q1, q2 = one - p1, P(2) + p1
    inv, c3 = one / p1, P(3) / q2
    z = np.zeros_like(p1)
    s = [[z, h * (one / q1), h * (P(4) / q1)],
         [h * inv, z, h * (P(3) / q1)],
         [h * (inv + c3), h * c3, z]]
  return np.array([[np.asarray(e, dtype=np.float64) for e in r] for r in s])


def _time_mean(v, case):
  """The kernel's time mean: float64 values added in group order."""
  v = v.reshape((case.nout, case.ngroup) + v.shape[1:])
  if case.ngroup == 1:
    return v[:, 0].astype(np.float32)
  acc = np.zeros((case.nout,) + v.shape[2:])
  cnt = np.zeros(acc.shape)
  for g in range(case.ngroup):
    x = v[:, g]
    if case.skipna:
      ok = ~np.isnan(x)
      acc = np.where(ok, acc + np.where(ok, x, 0.0), acc)
      cnt += ok
    else:
      acc = acc + x
  with np.errstate(all='ignore'):
    r = acc / cnt if case.skipna else acc / case.ngroup
  if case.skipna:
    r = np.where(cnt > 0, r, np.nan)
  return r.astype(np.float32)


def kernel_model(case):
  """The kernel's arithmetic: float32 [nout][nrow][ncol]."""
  fc = categories(case.f, case.dry, case.wet_at('f'))
  tc = categories(case.t, case.dry, case.wet_at('t'))
  S = scoring_matrix(case.p1)
  P = case.p1.dtype.type
  with np.errstate(all='ignore'):
    masked = ~(case.p1 < P(case.max_p1)) | ~(case.p1 > P(case.min_p1))
    v = np.zeros(case.f.shape)
    for a in range(3):
      for b in range(3):
        v = v + (fc[a] & tc[b]).astype(np.float64) * S[a, b]
  v[fc[3] | tc[3] | masked[None]] = np.nan
  return _time_mean(v, case)


def old_kernel_model(case):
  """The previous kernel: every operand cast to float32 on the host, the
  matrix formed in float64 from the float32 p1 and rounded once per entry,
  only the selected entries added, each step rounded to float32 before a
  float64 time mean."""
  f32 = lambda a: np.asarray(a).astype(np.float32)  # noqa: E731
  dry = float(np.float32(case.dry))
  fc = categories(f32(case.f), dry, f32(case.wet_at('f')))
  tc = categories(f32(case.t), dry, f32(case.wet_at('t')))
  p = f32(case.p1).astype(np.float64)
  with np.errstate(all='ignore'):
    z = np.zeros_like(p)
    S = np.array([[z, 0.5 / (1 - p), 2 / (1 - p)],
                  [0.5 / p, z, 1.5 / (1 - p)],
                  [0.5 * (1 / p + 3 / (2 + p)), 1.5 / (2 + p), z]])
    masked = (~(p < float(np.float32(case.max_p1))) |
              ~(p > float(np.float32(case.min_p1))))
    v = np.zeros(case.f.shape)
    for a in range(3):
      for b in range(3):
        v = v + np.where(fc[a] & tc[b], S[a, b], 0.0)
  v[fc[3] | tc[3] | masked[None]] = np.nan
  return _time_mean(v.astype(np.float32).astype(np.float64), case)


# ---- edges -------------------------------------------------------------------------
def _nb(x, dtype, direction):
  return np.nextafter(dtype.type(x), dtype.type(direction), dtype=dtype)


def _between32(x, c):
  """float64 `x` strictly between the float32 neighbours of float32(c), and
  not equal to c (compared in float64)."""
  c = np.asarray(c, dtype=np.float64)
  c32 = c.astype(np.float32)
  lo = np.nextafter(c32, np.float32(-np.inf)).astype(np.float64)
  hi = np.nextafter(c32, np.float32(np.inf)).astype(np.float64)
  return (x > lo) & (x < hi) & (x != c)


def _value_edges(side, x, wet, dry, p1ok):
  out = set()
  dt = x.dtype
  dx = dt.type(dry)
  if dt == F32:
    for e, v in (('below_dry', _nb(dx, dt, -np.inf)), ('at_dry', dx),
                 ('above_dry', _nb(dx, dt, np.inf))):
      if (x == v).any():
        out.add(e)
  if dt == wet.dtype == F32:
    for e, v in (('below_wet', np.nextafter(wet, np.float32(-np.inf))),
                 ('at_wet', wet), ('above_wet', np.nextafter(wet, np.float32(np.inf)))):
      if (np.isfinite(wet) & (x == v)).any():
        out.add(e)
  with np.errstate(all='ignore'):
    checks = {'pos_zero': (x == 0) & ~np.signbit(x),
              'neg_zero': (x == 0) & np.signbit(x),
              'negative': (x < 0) & np.isfinite(x), 'nan': np.isnan(x),
              'pos_inf': x == np.inf, 'neg_inf': x == -np.inf}
    d, l, h, n = categories(x, dry, wet)
    checks['no_category'] = ~(d | l | h | n)
    if dt == F64:
      xd = x.astype(np.float64)
      checks['f64_near_dry'] = _between32(xd, dry)
      checks['f64_near_wet'] = np.isfinite(wet) & _between32(
          xd, wet.astype(np.float64))
  out |= {e for e, m in checks.items() if (m & p1ok).any()}
  return {f'{side}_{e}' for e in out}


def reached_edges(case):
  """The edges the arrays of `case` reach."""
  out = set()
  P = case.p1.dtype.type
  with np.errstate(all='ignore'):
    p1ok = (case.p1 < P(case.max_p1)) & (case.p1 > P(case.min_p1))
  for side, x in (('f', case.f), ('t', case.t)):
    out |= _value_edges(side, x, case.wet_at(side), case.dry, p1ok)
  fc = categories(case.f, case.dry, case.wet_at('f'))
  tc = categories(case.t, case.dry, case.wet_at('t'))
  for a, ca in enumerate('dlh'):
    for b, cb in enumerate('dlh'):
      if (fc[a] & tc[b] & p1ok).any():
        out.add(f'cell_{ca}{cb}')
  if any(((c[0] & c[2]) & p1ok).any() for c in (fc, tc)):
    out.add('two_categories')
  wet = np.concatenate([case.wet_at('f'), case.wet_at('t')])
  w64 = wet.astype(np.float64)
  dry_w = np.float64(wet.dtype.type(case.dry))
  with np.errstate(all='ignore'):
    for e, m in (('wet_below_dry', w64 < dry_w), ('wet_eq_dry', w64 == dry_w),
                 ('wet_nan', np.isnan(w64)), ('wet_zero', w64 == 0),
                 ('wet_inf', w64 == np.inf),
                 ('wet_0.5_to_20mm', (w64 >= 0.5e-3) & (w64 <= 20e-3))):
      if m.any():
        out.add(e)
    if wet.dtype == F64:
      for x, w in ((case.f, case.wet_at('f')), (case.t, case.wet_at('t'))):
        if x.dtype == F32 and ((x == w.astype(np.float32)) &
                               (x.astype(np.float64) != w)).any():
          out.add('precip32_at_rounded_wet64')
  p1 = case.p1
  if p1.dtype == F32:
    for e, v in (('p1_at_min', P(case.min_p1)),
                 ('p1_below_min', _nb(case.min_p1, F32, -np.inf)),
                 ('p1_above_min', _nb(case.min_p1, F32, np.inf)),
                 ('p1_at_max', P(case.max_p1)),
                 ('p1_below_max', _nb(case.max_p1, F32, -np.inf)),
                 ('p1_above_max', _nb(case.max_p1, F32, np.inf))):
      if (p1 == v).any():
        out.add(e)
  else:
    p64 = p1.astype(np.float64)
    if _between32(p64, case.min_p1).any():
      out.add('p1_f64_near_min')
    if _between32(p64, case.max_p1).any():
      out.add('p1_f64_near_max')
  with np.errstate(all='ignore'):
    for e, m in (('p1_zero', p1 == 0), ('p1_one', p1 == 1),
                 ('p1_nan', np.isnan(p1)),
                 ('p1_masked_low', (p1 > 0) & (p1 <= P(case.min_p1))),
                 ('p1_masked_high', (p1 < 1) & (p1 >= P(case.max_p1)))):
      if m.any():
        out.add(e)
    pos = np.concatenate([case.f.ravel(), case.t.ravel()])
    if (pos == 0).mean() > 0.3:
      out.add('exact_zero')
    if ((pos > 0) & (pos < 1e-6)).any():
      out.add('tiny_positive')
    if ((pos < 0) & (pos > -1e-9)).any():
      out.add('small_negative')
  out.add('mix_' + '_'.join(
      '64' if a.dtype == F64 else '32'
      for a in (case.f, case.t, case.wet, case.p1)))
  out.add(f'ngroup{"1" if case.ngroup == 1 else "N"}_skipna{int(case.skipna)}')
  if case.ngroup > 1:
    g = (np.isnan(case.f) | np.isnan(case.t)).reshape(
        (case.nout, case.ngroup, -1)).all(axis=1)
    if (g & p1ok.reshape(1, -1)).any():
      out.add('all_nan_series')
  if case.wet.shape[2] > case.ncol:
    out.add('wet_row_stride')
  if case.nout >= 1000:
    out.add('many_outputs')
  if (case.nrow * case.ncol) % 256:
    out.add('partial_block')
  return out


# ---- realistic cases -----------------------------------------------------------
def realistic_precip(rs, shape, dtype):
  """24-hour precipitation in metres: 40-60 % exact zeros (the share varies
  with longitude), gamma-distributed wet amounts, tiny positive values and
  small negatives as packed reanalysis data has."""
  zero_share = 0.5 + 0.1 * np.sin(np.linspace(0, 4 * np.pi, shape[-1]))
  u = rs.uniform(size=shape)
  x = rs.gamma(0.7, 4e-3, size=shape)
  x = np.where(u < zero_share, 0.0, x)
  tiny = rs.uniform(size=shape) < 0.04
  x = np.where(tiny, 10 ** rs.uniform(-9, -6, size=shape), x)
  neg = rs.uniform(size=shape) < 0.02
  x = np.where(neg, -1e-10 * rs.uniform(0.5, 2.0, size=shape), x)
  return x.astype(dtype)


def p1_profile(lat, lon, rs, dtype):
  """The climatological dry fraction on a latitude profile: below 0.1 in the
  wet tropics, above 0.85 over the subtropical deserts, mid values elsewhere,
  with cell-to-cell noise."""
  la = np.asarray(lat, dtype=np.float64)[:, None]
  base = (0.55 - 0.5 * np.exp(-(la / 8.0) ** 2) +
          0.4 * np.exp(-((np.abs(la) - 25.0) / 7.0) ** 2))
  lo = np.deg2rad(np.asarray(lon, dtype=np.float64))[None, :]
  p = base + 0.05 * np.sin(3 * lo) + 0.03 * rs.standard_normal(
      (la.size, lo.size))
  return np.clip(p, 0.01, 0.99).astype(dtype)


def wet_climatology(lat, lon, ndays, rs, dtype):
  """Wet thresholds of 0.5 to 20 mm, in metres, for `ndays` days:
  [ndays][nlat][nlon]."""
  la = np.asarray(lat, dtype=np.float64)[:, None]
  base = 2e-3 + 12e-3 * np.exp(-(la / 15.0) ** 2)
  lo = np.deg2rad(np.asarray(lon, dtype=np.float64))[None, :]
  days = np.arange(ndays)[:, None, None]
  w = base * (1 + 0.3 * np.sin(2 * lo + days / 9.0)) * rs.uniform(
      0.8, 1.2, (ndays, la.size, lo.size))
  return np.clip(w, 0.5e-3, 20e-3).astype(dtype)


def leap_year_lookup(inits, nlead):
  """Day-of-year slab (0-based, 366 days) of every (init, lead) valid time,
  leads of 1..nlead days."""
  vt = inits[:, None] + np.arange(1, nlead + 1)[None, :] * DAY
  return (pd.DatetimeIndex(vt.ravel()).dayofyear.values - 1).reshape(vt.shape)


def _realistic(name, lat, lon, inits, nlead, dtypes, ngroup_init, skipna,
               seed):
  rs = np.random.RandomState(seed)
  fdt, tdt, wdt, pdt = dtypes
  doy = leap_year_lookup(inits, nlead)   # [init][lead]
  days, inv = np.unique(doy, return_inverse=True)
  inv = inv.reshape(doy.shape)
  wet = wet_climatology(lat, lon, days.size, rs, wdt)
  # fields ordered (lead, init): the init times are the averaged group
  shape = (nlead, len(inits), lat.size, lon.size)
  f = realistic_precip(rs, shape, fdt)
  t = realistic_precip(rs, shape, tdt)
  slab = inv.T.reshape(-1)
  ngroup = len(inits) if ngroup_init else 1
  edges = {'exact_zero', 'tiny_positive', 'small_negative', 'wet_0.5_to_20mm',
           'p1_masked_low', 'p1_masked_high', 'partial_block',
           'mix_' + '_'.join('64' if d == F64 else '32' for d in dtypes),
           f'ngroup{"N" if ngroup > 1 else "1"}_skipna{int(skipna)}'}
  edges |= {f'cell_{a}{b}' for a in 'dlh' for b in 'dlh'}
  return Case(name, frozenset(edges), f.reshape((-1,) + f.shape[2:]),
              t.reshape((-1,) + t.shape[2:]), wet,
              p1_profile(lat, lon, rs, pdt), slab, slab, ngroup, skipna)


LAT_1P5 = np.linspace(-90, 90, 121)
LON_1P5 = np.arange(240) * 1.5
LAT_BAND = np.arange(97) * 0.25 - 2.0      # 2 S (wet) to 22 N (desert)
LON_025 = np.arange(1440) * 0.25
LEAP_INITS = np.array(['2024-02-22', '2024-12-27'], dtype='datetime64[ns]')
LEAP_INITS4 = np.array(['2024-02-20', '2024-02-25', '2024-12-24',
                        '2024-12-29'], dtype='datetime64[ns]')


def realistic_cases():
  """The realistic family (REALISTIC_NAMES)."""
  A32 = (F32,) * 4
  return [
      _realistic('era5_1p5_f32', LAT_1P5, LON_1P5, LEAP_INITS4, 10, A32, False,
                 False, 901),
      _realistic('era5_1p5_f32_mean', LAT_1P5, LON_1P5, LEAP_INITS4, 10, A32,
                 True, False, 902),
      _realistic('era5_1p5_f64_mean_skipna', LAT_1P5, LON_1P5, LEAP_INITS4, 10,
                 (F64,) * 4, True, True, 903),
      _realistic('band_025_f32', LAT_BAND, LON_025, LEAP_INITS, 3, A32, False,
                 False, 904),
      _realistic('band_025_f64_precip', LAT_BAND, LON_025, LEAP_INITS, 3,
                 (F64, F32, F32, F32), True, True, 905),
  ]


# ---- edge cases ---------------------------------------------------------------------
def _edge_values(dry, wet):
  """float32 values at the category edges of `dry` / `wet`: one ulp below, at
  and one ulp above each, a light value, +-0, a negative, NaN, +-inf."""
  d32, w32 = np.float32(dry), np.float32(wet)
  dn = lambda v: np.nextafter(v, np.float32(-np.inf))  # noqa: E731
  up = lambda v: np.nextafter(v, np.float32(np.inf))   # noqa: E731
  return np.array([dn(d32), d32, up(d32), np.float32(1e-3), dn(w32), w32,
                   up(w32), 0.0, -0.0, -1e-3, np.nan, np.inf, -np.inf],
                  dtype=np.float32)


def _pairs(values_f, values_t):
  """f[r, c] = values_f[r], t[r, c] = values_t[c]."""
  nr, nc = values_f.size, values_t.size
  return (np.broadcast_to(values_f[:, None], (nr, nc)).copy(),
          np.broadcast_to(values_t[None, :], (nr, nc)).copy())


def _case(name, edges, f, t, wet, p1, wf=None, wt=None, **kw):
  f = f if f.ndim == 3 else f[None]
  t = t if t.ndim == 3 else t[None]
  wet = wet if wet.ndim == 3 else wet[None]
  n = f.shape[0]
  wf = np.zeros(n, np.int64) if wf is None else np.asarray(wf, np.int64)
  wt = wf if wt is None else np.asarray(wt, np.int64)
  return Case(name, frozenset(edges), f, t, wet, p1, wf, wt, **kw)


def edge_cases():
  dry = DRY_MM / 1000.0
  wet = 4e-3
  out = []
  # every (forecast, truth) pair of edge values against one wet threshold
  v = _edge_values(dry, wet)
  f, t = _pairs(v, v)
  p1 = np.full(f.shape, 0.4, np.float32)
  wetf = np.full(f.shape, wet, np.float32)
  sides = [f'{s}_{e}' for s in 'ft' for e in (
      'below_dry', 'at_dry', 'above_dry', 'below_wet', 'at_wet', 'above_wet',
      'pos_zero', 'neg_zero', 'negative', 'nan', 'pos_inf', 'neg_inf',
      'no_category')]
  out.append(_case('value_edges', set(sides) | set(CELL_EDGES) |
                   {'mix_32_32_32_32', 'ngroup1_skipna0', 'partial_block'},
                   f, t, wetf, p1))
  # wet below the dry threshold (two categories), equal to it, NaN, 0, inf:
  # column block k has wet W[k]; the values include one between wet and dry
  W = np.array([1e-4, dry, np.nan, 0.0, np.inf], dtype=np.float32)
  v2 = np.concatenate([v, np.array([1.5e-4], np.float32)])
  f, t = _pairs(v2, v2)
  f, t = np.tile(f, (1, W.size)), np.tile(t, (1, W.size))
  wetf = np.repeat(W, v2.size)[None, :].repeat(v2.size, axis=0)
  p1 = np.full(f.shape, 0.3, np.float32)
  out.append(_case('wet_edges', {'wet_below_dry', 'wet_eq_dry', 'wet_nan',
                                 'wet_zero', 'wet_inf', 'two_categories',
                                 'partial_block'}, f, t, wetf, p1))
  # p1 at and next to the mask bounds, 0, 1, NaN: a column per p1, a row per
  # table cell (and NaN)
  P = np.array([np.float32(0.1), _nb(0.1, F32, -np.inf), _nb(0.1, F32, np.inf),
                np.float32(0.85), _nb(0.85, F32, -np.inf),
                _nb(0.85, F32, np.inf), 0.0, 1.0, np.nan, 0.5, 0.05, 0.95],
               dtype=np.float32)
  reps = np.array([0.0, 1e-3, 0.01, np.nan], np.float32)   # dry, light, heavy
  rf = np.repeat(reps, reps.size)
  rt = np.tile(reps, reps.size)
  f = np.broadcast_to(rf[:, None], (rf.size, P.size)).copy()
  t = np.broadcast_to(rt[:, None], (rt.size, P.size)).copy()
  p1 = np.broadcast_to(P[None, :], f.shape).copy()
  wetf = np.full(f.shape, wet, np.float32)
  out.append(_case('p1_edges', {'p1_at_min', 'p1_below_min', 'p1_above_min',
                                'p1_at_max', 'p1_below_max', 'p1_above_max',
                                'p1_zero', 'p1_one', 'p1_nan',
                                'p1_masked_low', 'p1_masked_high'},
                   f, t, wetf, p1))
  return out


def _f64_near(c, n, rs):
  """n float64 values strictly between the float32 neighbours of float32(c),
  none equal to c: float32(c) itself, values a few float64 ulps and a few
  parts in 1e9 either side of c, and uniform draws from the open interval."""
  c32 = np.float32(c)
  lo = float(np.nextafter(c32, np.float32(-np.inf)))
  hi = float(np.nextafter(c32, np.float32(np.inf)))
  fixed = [float(c32), float(np.nextafter(c, 1.0)),
           float(np.nextafter(c, -1.0)), c * (1 + 1e-9), c * (1 - 1e-9),
           (lo + c) / 2, (c + hi) / 2, float(np.nextafter(hi, -1.0)),
           float(np.nextafter(lo, 1.0))]
  x = np.concatenate([fixed, rs.uniform(lo, hi, max(n - len(fixed), 0))])[:n]
  x = x[(x > lo) & (x < hi) & (x != c)]
  return x


def float64_cases():
  rs = np.random.RandomState(77)
  dry = DRY_MM / 1000.0
  wet64 = 0.0021234567891
  wet32 = np.float32(3.1e-3)
  out = []
  # float64 forecast and truth near the dry threshold and near a float32 /
  # float64 wet threshold; the other side takes a value of each category
  near = np.concatenate([_f64_near(dry, 24, rs),
                         _f64_near(float(wet32), 24, rs)])
  other = np.array([0.0, 1e-3, 0.01, -0.0, dry], np.float64)
  f, t = _pairs(near, other)
  p1 = np.full(f.shape, 0.45, np.float64)
  wet = np.full(f.shape, wet32, np.float32)
  out.append(_case('f64_forecast_near_thresholds',
                   {'f_f64_near_dry', 'f_f64_near_wet'}, f, t, wet,
                   p1.astype(np.float32)))
  out.append(_case('f64_truth_near_thresholds',
                   {'t_f64_near_dry', 't_f64_near_wet', 'mix_64_64_64_64'},
                   t.T.copy(), f.T.copy(), wet.T.astype(np.float64),
                   p1.T.copy()))
  # a float64 forecast against float32 truth and wet
  ff = np.concatenate([_f64_near(dry, 30, rs), _f64_near(float(wet32), 30, rs)])
  tt = np.array([0.0, 1e-3, 0.01], np.float32)
  f, t = _pairs(ff, tt)
  out.append(_case('f64_forecast_f32_truth_wet',
                   {'mix_64_32_32_32', 'f_f64_near_dry', 'f_f64_near_wet'},
                   f, t, np.full(f.shape, wet32, np.float32),
                   np.full(f.shape, 0.3, np.float32)))
  # float32 precipitation against a float64 wet threshold that float32
  # cannot hold: its float32 rounding and neighbours on both sides
  w32 = np.float32(wet64)
  vals = np.array([np.nextafter(w32, np.float32(0)), w32,
                   np.nextafter(w32, np.float32(1)), 0.0, 1e-3,
                   np.float32(dry)], np.float32)
  f, t = _pairs(vals, vals)
  out.append(_case('f32_precip_f64_wet', {'mix_32_32_64_32',
                                          'precip32_at_rounded_wet64'},
                   f, t, np.full(f.shape, wet64, np.float64),
                   np.full(f.shape, 0.6, np.float32)))
  # float64 p1 strictly between the float32 neighbours of 0.1 and 0.85
  P = np.concatenate([_f64_near(0.1, 20, rs), _f64_near(0.85, 20, rs)])
  reps = np.array([0.0, 1e-3, 0.01], np.float32)
  rf, rt = np.repeat(reps, 3), np.tile(reps, 3)
  f = np.broadcast_to(rf[:, None], (rf.size, P.size)).copy()
  t = np.broadcast_to(rt[:, None], (rt.size, P.size)).copy()
  p1 = np.broadcast_to(P[None, :], f.shape).copy()
  out.append(_case('f64_p1_near_bounds', {'mix_32_32_32_64',
                                          'p1_f64_near_min',
                                          'p1_f64_near_max'},
                   f, t, np.full(f.shape, 4e-3, np.float32), p1))
  return out


def geometry_cases():
  rs = np.random.RandomState(5)
  out = []
  lat = np.linspace(-60, 60, 17)
  lon = np.arange(45) * 8.0
  for skipna in (False, True):
    # ngroup > 1 with an all-NaN series in some cells
    ng = 6
    f = realistic_precip(rs, (3 * ng, 17, 45), F32)
    t = realistic_precip(rs, (3 * ng, 17, 45), F32)
    f[:, 3, 4:9] = np.nan
    t[::2, 5, 10:12] = np.nan
    f[1::2, 5, 10:12] = np.nan
    wet = wet_climatology(lat, lon, 4, rs, F32)
    pad = np.full((4, 17, 64), np.nan, np.float32)   # its own row stride
    pad[:, :, :45] = wet
    p1 = np.clip(p1_profile(lat, lon, rs, F32), 0.12, 0.8)
    wf = rs.randint(0, 4, 3 * ng)
    out.append(_case(f'grouped_skipna{int(skipna)}',
                     {f'ngroupN_skipna{int(skipna)}', 'all_nan_series',
                      'wet_row_stride'}, f, t, pad, p1, wf,
                     rs.randint(0, 4, 3 * ng), ngroup=ng, skipna=skipna))
  # ngroup 1 with skipna set (compute over a single init time)
  f = realistic_precip(rs, (2, 17, 45), F32)
  t = realistic_precip(rs, (2, 17, 45), F32)
  out.append(_case('single_skipna1', {'ngroup1_skipna1'}, f, t,
                   wet_climatology(lat, lon, 2, rs, F32),
                   p1_profile(lat, lon, rs, F32), [0, 1], [1, 0], skipna=True))
  # many outputs on a small grid
  n = 1500
  f = realistic_precip(rs, (2 * n, 3, 7), F32)
  t = realistic_precip(rs, (2 * n, 3, 7), F32)
  out.append(_case('many_outputs', {'many_outputs', 'ngroupN_skipna0'}, f, t,
                   wet_climatology(np.array([-10., 0., 10.]),
                                   np.arange(7) * 50., 3, rs, F32),
                   np.full((3, 7), 0.5, np.float32), rs.randint(0, 3, 2 * n),
                   rs.randint(0, 3, 2 * n), ngroup=2))
  return out


def raw_cases():
  return (realistic_cases() + edge_cases() + float64_cases() +
          geometry_cases())


REALISTIC_NAMES = ('era5_1p5_f32', 'era5_1p5_f32_mean',
                   'era5_1p5_f64_mean_skipna', 'band_025_f32',
                   'band_025_f64_precip')


# ---- lookup cases (operators) -----------------------------------------------------
@dataclasses.dataclass
class LookupCase:
  name: str
  edges: frozenset
  inits: np.ndarray          # datetime64[ns]
  leads: np.ndarray          # timedelta64[ns]
  hours: np.ndarray          # climatology `hour` labels
  days: np.ndarray           # climatology `dayofyear` labels, in their order
  raises: bool = False

  def valid_times(self):
    return self.inits[:, None] + self.leads[None, :]


def run_entry(ctx, case, upload):
  """`ctx.seeps_maps` on `case`: float32 [nout][nrow][ncol].  `upload(array)`
  returns the device address of a copy of the array (kept alive by the
  caller)."""
  from weatherbench2_b200 import _lib  # pylint: disable=import-outside-toplevel
  code = lambda a: _lib.F64 if a.dtype == F64 else _lib.F32  # noqa: E731
  slab = case.nrow * case.ncol
  wslab = case.nrow * case.wet.shape[2]
  idx = np.arange(case.nfield, dtype=np.int64)
  out_shape = (case.nout, case.nrow, case.ncol)
  out = ctx.malloc(int(np.prod(out_shape)) * 4)
  try:
    ctx.seeps_maps(upload(case.f), upload(case.t), upload(case.wet),
                   upload(case.p1), case.nout, case.ngroup, idx * slab,
                   idx * slab, case.wf.astype(np.int64) * wslab,
                   case.wt.astype(np.int64) * wslab, case.nrow, case.ncol,
                   case.ncol, case.wet.shape[2], case.dry, case.min_p1,
                   case.max_p1, case.skipna, out, f_dtype=code(case.f),
                   t_dtype=code(case.t), wet_dtype=code(case.wet),
                   p1_dtype=code(case.p1))
    return ctx.from_device(out, out_shape, np.float32)
  finally:
    ctx.free(out)


LOOKUP_EDGES = frozenset({'feb29', 'dec31_leap', 'dec31_nonleap',
                          'year_boundary', 'hourly6', 'hourly24',
                          'unsorted_doy', 'subset_doy', 'missing_hour'})


def lookup_cases():
  D = lambda *s: np.array(s, dtype='datetime64[ns]')  # noqa: E731
  days = np.arange(1, 367)
  rs = np.random.RandomState(11)
  return [
      LookupCase('leap_year_6hourly', frozenset({'feb29', 'dec31_leap',
                                                 'year_boundary', 'hourly6'}),
                 D('2024-02-27T06', '2024-12-30T12'),
                 np.arange(0, 13) * 6 * HOUR, np.array([0, 6, 12, 18]), days),
      LookupCase('non_leap_daily', frozenset({'dec31_nonleap', 'hourly24',
                                              'year_boundary'}),
                 D('2022-12-29', '2023-12-28', '2023-02-26'),
                 np.arange(1, 6) * DAY, np.array([0]), days),
      LookupCase('unsorted_subset_doy', frozenset({'unsorted_doy',
                                                   'subset_doy', 'feb29',
                                                   'hourly24'}),
                 D('2024-02-26', '2024-03-01'), np.arange(0, 5) * DAY,
                 np.array([0]), rs.permutation(np.arange(50, 70))),
      LookupCase('missing_hour', frozenset({'missing_hour'}),
                 D('2024-01-10'), np.array([0, 6]) * HOUR, np.array([0, 12]),
                 days, raises=True),
  ]


def lookup_reached(case):
  vt = pd.DatetimeIndex(case.valid_times().ravel())
  out = set()
  if ((vt.month == 2) & (vt.day == 29)).any():
    out.add('feb29')
  dec31 = (vt.month == 12) & (vt.day == 31)
  if (dec31 & vt.is_leap_year).any():
    out.add('dec31_leap')
  if (dec31 & ~vt.is_leap_year).any():
    out.add('dec31_nonleap')
  if len(set(vt.year)) > 1:
    out.add('year_boundary')
  if set(vt.hour) >= {0, 6, 12, 18} and set(case.hours) == {0, 6, 12, 18}:
    out.add('hourly6')
  if set(vt.hour) == {0} and list(case.hours) == [0]:
    out.add('hourly24')
  if (np.diff(case.days) < 0).any():
    out.add('unsorted_doy')
  if case.days.size < 366:
    out.add('subset_doy')
  if not set(vt.hour) <= set(case.hours):
    out.add('missing_hour')
  return out


def lookup_positions(case):
  """(hour index, dayofyear index) of every valid time, found label by label;
  KeyError for a label the climatology lacks."""
  vt = case.valid_times()
  stamps = pd.DatetimeIndex(vt.ravel())
  hi, di = [], []
  for h, d in zip(stamps.hour, stamps.dayofyear):
    if h not in case.hours or d not in case.days:
      raise KeyError((h, d))
    hi.append(int(np.flatnonzero(case.hours == h)[0]))
    di.append(int(np.flatnonzero(case.days == d)[0]))
  return np.reshape(hi, vt.shape), np.reshape(di, vt.shape)


def lookup_data(case, dtypes=(F32, F32, F32, F32), nlat=19, nlon=36, seed=0):
  """(forecast arrays, climatology arrays, coords) of `case`:
  f / t [init][lead][lat][lon], wet / dry fraction [hour][day][lat][lon]."""
  rs = np.random.RandomState(seed)
  fdt, tdt, wdt, pdt = dtypes
  lat = np.linspace(-90, 90, nlat)
  lon = np.arange(nlon) * (360.0 / nlon)
  shape = (case.inits.size, case.leads.size, nlat, nlon)
  f = realistic_precip(rs, shape, fdt)
  t = realistic_precip(rs, shape, tdt)
  nh, nd = case.hours.size, case.days.size
  wet = wet_climatology(lat, lon, nh * nd, rs, wdt).reshape(
      (nh, nd, nlat, nlon))
  frac = np.clip(p1_profile(lat, lon, rs, np.float64)[None, None] +
                 0.05 * rs.standard_normal((nh, nd, nlat, nlon)), 0, 1)
  frac[0, 0, 2, :5] = np.nan
  return (dict(f=f, t=t, wet=wet, frac=frac.astype(pdt)),
          dict(lat=lat, lon=lon))


def lookup_datasets(case, arrays, coords, to=None):
  """xarray_lite datasets (forecast, truth, climatology); `to` converts the
  forecast / truth arrays (e.g. to CUDA tensors)."""
  from weatherbench2_b200 import xarray_lite as xl  # pylint: disable=import-outside-toplevel
  conv = to or (lambda a: a)
  dims = ('init_time', 'lead_time', 'latitude', 'longitude')
  c = dict(init_time=case.inits, lead_time=case.leads,
           latitude=coords['lat'], longitude=coords['lon'],
           valid_time=(('init_time', 'lead_time'), case.valid_times()))
  fds = xl.Dataset({NAME: (dims, conv(arrays['f']))}, c)
  tds = xl.Dataset({NAME: (dims, conv(arrays['t']))}, c)
  cdims = ('hour', 'dayofyear', 'latitude', 'longitude')
  clim = xl.Dataset({NAME + '_seeps_threshold': (cdims, arrays['wet']),
                     NAME + '_seeps_dry_fraction': (cdims, arrays['frac'])},
                    dict(hour=case.hours, dayofyear=case.days,
                         latitude=coords['lat'], longitude=coords['lon']))
  return fds, tds, clim


def lookup_reference(case, arrays, skipna=None, min_p1=0.1, max_p1=0.85):
  """float64 maps [init][lead][lat][lon] (skipna None), or their mean over
  init_time, of the reference on `case`."""
  hi, di = lookup_positions(case)
  wet = arrays['wet'][hi, di]
  ctx = _quiet()
  try:
    p1 = np.nanmean(arrays['frac'], axis=(0, 1))
    with np.errstate(all='ignore'):
      pt = orc.seeps_pointwise(arrays['f'], arrays['t'], wet, wet, p1, DRY_MM,
                               min_p1, max_p1)
    if skipna is None:
      return pt
    return orc.time_mean(pt, ('init_time', 'lead_time', 'lat', 'lon'),
                         skipna=skipna, avg_dim='init_time')[0]
  finally:
    ctx.__exit__(None, None, None)

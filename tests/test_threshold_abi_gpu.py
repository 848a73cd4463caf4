"""The threshold and Gaussian-forecast kernels (csrc/threshold_metrics.cu)
called through `_lib.Context` directly, cell by cell, on the seeded cases of
threshold_cases.py, against the oracle's float64 point-wise scores.

Reached here and nowhere else: members and truth at the float32 bracket
[lo, hi] of a float64 threshold and next to it, thresholds whose two float64
roundings give a float32 number that one rounding (fma) would not, thresholds
beyond float32 range, warps that take the one-comparison shortcut or the
two-comparison path on purpose, 11 member counts from 1 to 5000 in two
layouts, every pass mix of 4 / 2 / 1 thresholds, Gaussian offsets from 0 to
+-inf across the float32 / float64 switch and the `1 - cdf` saturation, std of
0, 1e-30, inf and NaN, row segments longer than the prefetch ring, regions,
zero-weight cells holding NaN, and every argument error of the three entries."""
import numpy as np
import pytest
from scipy import special

import threshold_cases as tc
from threshold_cases import F32, F64, U

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def ctx():
  from weatherbench2_b200 import _lib
  return _lib.default_context(0)


def _dev(a):
  import torch
  return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _ptr(a):
  return None if a is None else a.data_ptr()


def _thr_dev(case):
  a, b = case.thr_buffers() if case.nq else (None, None)
  return (None if a is None else _dev(a)), (None if b is None else _dev(b))


def ens_point(ctx, case, skipna, z=None):
  """[nq][ncell][8] of wb2_ens_threshold_metrics, one field per cell."""
  import torch
  n = case.ncell
  x, t = _dev(case.x_buffer()), _dev(case.t)
  a, b = _thr_dev(case)
  off_a, off_b = case.off_thr()
  out = torch.full((n, case.nq, 1, 8), 7.0, dtype=torch.float64, device='cuda')
  ctx.ens_threshold_metrics(
      x.data_ptr(), t.data_ptr(), case.nmember, case.member_stride(),
      case.off_x(), np.arange(n, dtype=np.int64), case.nq, a.data_ptr(), off_a,
      _ptr(b), off_b, case.z if z is None else z, tc.geometry_1x1(), skipna,
      out.data_ptr())
  return out.cpu().numpy()[:, :, 0].transpose(1, 0, 2)


def ens_maps(ctx, case, stat, skipna):
  """[nq][ncell] of wb2_ens_threshold_maps: one map, ngroup = 1, cells on
  consecutive lanes (member-major layout)."""
  import torch
  assert not case.interleaved
  n = case.ncell
  x, t = _dev(case.x_buffer()), _dev(case.t)
  a, b = _thr_dev(case)
  gq = b is not None
  off_a = (np.zeros(1, np.int64) if gq
           else np.arange(case.nq, dtype=np.int64) * n)
  out = torch.full((case.nq, 1, n), 7.0, device='cuda')
  ctx.ens_threshold_maps(
      x.data_ptr(), t.data_ptr(), case.nmember, n, 1, 1,
      np.zeros(1, np.int64), np.zeros(1, np.int64), case.nq, a.data_ptr(),
      off_a, _ptr(b), np.zeros(1, np.int64) if gq else None, case.z, 1, n, n,
      stat, skipna, out.data_ptr())
  return out.cpu().numpy()[:, 0]


def gauss_point(ctx, case, skipna=False):
  """[max(nq, 1)][ncell][8] of wb2_gaussian_metrics, one field per cell."""
  import torch
  n = case.ncell
  m, s, t = _dev(case.mean), _dev(case.std), _dev(case.t)
  a, b = _thr_dev(case)
  off_a, off_b = case.off_thr() if case.nq else (None, None)
  c = np.arange(n, dtype=np.int64)
  out = torch.full((n, max(case.nq, 1), 1, 8), 7.0, dtype=torch.float64,
                   device='cuda')
  ctx.gaussian_metrics(m.data_ptr(), s.data_ptr(), t.data_ptr(), c, c, c,
                       case.nq, _ptr(a), off_a, _ptr(b), off_b, case.z,
                       tc.geometry_1x1(), skipna, out.data_ptr())
  return out.cpu().numpy()[:, :, 0].transpose(1, 0, 2)


def assert_same_specials(got, want, what):
  """Identical NaN, +inf and -inf patterns."""
  for f in (np.isnan, np.isposinf, np.isneginf):
    bad = f(got) != f(want)
    assert not bad.any(), (f'{what}: {f.__name__} differs at {np.argwhere(bad)[:5]}'
                           f' got {got[bad][:5]} want {want[bad][:5]}')


def assert_within(got, want, bound, what):
  ok = np.isfinite(got) & np.isfinite(want)
  err = np.abs(got - want)
  bad = ok & ~(err <= bound)
  assert not bad.any(), (f'{what}: {bad.sum()} cells out of bound, e.g. '
                         f'{np.argwhere(bad)[:3]} got {got[bad][:3]} want '
                         f'{want[bad][:3]} bound {np.asarray(bound * np.ones_like(got))[bad][:3]}')


# -- ensemble: point-wise values ---------------------------------------------------
def check_ens(got, case, skipna, what):
  """got [nq][ncell][4] point values against the oracle and the float32
  emulation of Brier / RPS."""
  want = case.oracle(skipna)
  m = case.nmember
  for k, name in enumerate(('brier', 'debiased', 'ignorance', 'rps')):
    assert_same_specials(got[..., k], want[..., k], f'{what} {name}')
  b32, r32, _ = tc.ens_emulate(case, skipna)
  if m <= 1551:
    # the Newton-step quotient is the IEEE quotient here: bit-exact
    np.testing.assert_array_equal(got[..., 0], b32.astype(F64), f'{what} brier')
    np.testing.assert_array_equal(got[..., 3], r32.astype(F64), f'{what} rps')
  # Brier / RPS: (p - [ind])^2 with p = c / n within one ulp (2u relative)
  # and one rounding of the difference and of the square
  for k in (0, 3):
    d = np.sqrt(np.abs(want[..., k]))
    e = 2 * U + U * d
    assert_within(got[..., k], want[..., k], 2 * d * e + e * e + 2 * U * want[..., k],
                  f'{what} stat {k}')
  # ignorance: -logf(c / M): the quotient's 2u plus one ulp of the result
  assert_within(got[..., 2], want[..., 2], 2 * U + 2 * U * np.abs(want[..., 2]),
                f'{what} ignorance')
  # debiased: brier - var / M.  The Brier part carries the bound above; var =
  # (c q1^2 + (n - c) p^2) / (n - 1) takes p and q1 = 1 - p with 2u absolute
  # error each, so var is within 4u n / (n - 1) <= 8u plus 4u var of its
  # value, and var / M within (8u + 4u var) / M plus one rounding
  b0 = want[..., 0]
  d0 = np.sqrt(np.abs(b0))
  e0 = 2 * U + U * d0
  var_m = np.abs(b0 - want[..., 1])
  assert_within(got[..., 1], want[..., 1],
                2 * d0 * e0 + e0 * e0 + 2 * U * b0 + 8 * U / m + 6 * U * var_m
                + U * np.abs(want[..., 1]) + 2.0 ** -149,
                f'{what} debiased')


def _point(case, got):
  """Point values from the raw sums: with skipna a NaN score leaves sum 0 and
  weight 0, so the value is NaN wherever the weight sum is 0."""
  return np.where(got[..., 4:] == 0, np.nan, got[..., :4])


@pytest.mark.parametrize('skipna', [False, True])
def test_bracket_m8_is_bit_equal_to_the_oracle(ctx, skipna):
  """M = 8: every probability and square is exact, so the kernel's Brier and
  RPS part equal the oracle's float64 values bit for bit, and the counts
  they imply are the exact #{x > thr} and #{x < thr}."""
  for case in tc.bracket_cases():
    raw = ens_point(ctx, case, skipna)
    got = _point(case, raw)
    want = case.oracle(skipna)
    check_ens(got, case, skipna, case.name)
    np.testing.assert_array_equal(got[..., 0], want[..., 0], case.name)
    np.testing.assert_array_equal(got[..., 3], want[..., 3], case.name)
    c_gt, c_lt = case.counts()
    tp = (case.t.astype(F64) > case.thresholds()).astype(F64)
    tl = (case.t.astype(F64) < case.thresholds()).astype(F64)
    fin = ~np.isnan(got[..., 0])
    imp_gt = 8 * np.abs(tp - np.sqrt(got[..., 0]))
    imp_lt = 8 * np.abs(tl - np.sqrt(got[..., 3]))
    np.testing.assert_array_equal(imp_gt[fin], c_gt[fin])
    np.testing.assert_array_equal(imp_lt, c_lt)
    # weight sums: 1, or 0 where skipna drops a NaN score
    for k in range(4):
      w = np.where(skipna & np.isnan(want[..., k]), 0.0, 1.0)
      np.testing.assert_array_equal(raw[..., 4 + k], w)
    for stat in range(4):
      mp = ens_maps(ctx, case, stat, skipna).astype(F64)
      pt = got[..., stat]
      assert_same_specials(mp, want[..., stat], f'maps stat {stat}')
      if stat in (0, 3):
        np.testing.assert_array_equal(mp, pt)
      else:
        fin = np.isfinite(mp)
        np.testing.assert_allclose(mp[fin], pt[fin], rtol=4 * U,
                                   atol=2.0 ** -149)


def _all_ens_cases():
  return (tc.field_cases() + tc.member_count_cases() +
          tc.threshold_count_cases())


@pytest.mark.parametrize('skipna', [False, True])
@pytest.mark.parametrize('case', _all_ens_cases(), ids=lambda c: c.name)
def test_ensemble_point_values(ctx, case, skipna):
  got = ens_point(ctx, case, skipna)
  check_ens(_point(case, got), case, skipna, case.name)
  if not case.interleaved:
    for stat in range(4):
      mp = ens_maps(ctx, case, stat, skipna).astype(F64)
      pt = _point(case, got)[..., stat]
      assert_same_specials(mp, pt, f'maps stat {stat}')
      fin = np.isfinite(mp)
      np.testing.assert_allclose(mp[fin], pt[fin], rtol=4 * U,
                                 atol=2.0 ** -149)


def test_shortcut_and_two_comparison_paths_agree_bit_for_bit(ctx):
  """A lane's scores do not depend on which path its warp took."""
  case, kinds = tc.warp_cases()
  strict = tc.warp_strictness(case)
  assert list(strict[0]) == [k == 'strict' or k == 'lastpass' for k in kinds]
  assert not strict[1].any()  # threshold 4 is a float32 number everywhere
  for stat in range(4):
    mp = ens_maps(ctx, case, stat, False).reshape(case.nq, -1, 32)
    for w, kind in enumerate(kinds):
      ref = mp[:, 0]
      lanes = np.arange(32) != 5 if kind == 'onelane' else slice(None)
      np.testing.assert_array_equal(mp[:, w, lanes], ref[:, lanes],
                                    f'stat {stat} warp {w} ({kind})')
  check_ens(_point(case, ens_point(ctx, case, False)), case, False, 'warps')


@pytest.mark.parametrize('form', ['gauss', 'field'])
def test_each_threshold_is_the_same_in_every_pass(ctx, form):
  """nq = 7 runs as passes of 4, 2 and 1; each threshold alone as a pass of
  1.  Launch counts follow the pass mix."""
  case = [c for c in tc.threshold_count_cases() if c.name == f'nq7_{form}'][0]
  before = ctx.launch_count
  full = ens_point(ctx, case, False)
  assert ctx.launch_count - before == 3 + 1
  before = ctx.launch_count
  maps = ens_maps(ctx, case, 3, False)
  assert ctx.launch_count - before == 3
  for k in range(7):
    one = tc.Case(case.name, 'ens', case.t, 1,
                  case.thr_a if form == 'gauss' else case.thr_a[k:k + 1],
                  case.thr_b, None if case.z is None else case.z[k:k + 1],
                  members=case.members)
    alone = ens_point(ctx, one, False)[0]
    # Brier, ignorance and RPS part (and every weight sum) bit for bit; the
    # debiased Brier's brier - var / M is contracted into fused multiply-adds
    # differently per pass width, so it may move by one float32 ulp
    for st in (0, 2, 3, 4, 5, 6, 7):
      np.testing.assert_array_equal(alone[:, st], full[k][:, st], f'{k} {st}')
    ulp = np.spacing(np.abs(full[k][:, 1]).astype(F32)).astype(F64)
    assert (np.abs(alone[:, 1] - full[k][:, 1]) <= ulp).all()
    np.testing.assert_array_equal(ens_maps(ctx, one, 3, False)[0], maps[k])


# -- Gaussian: point-wise values in two tiers -----------------------------------------
def gauss_reference(case):
  """Tier 1 (the kernel's float32 z, reference formulas in float64) and tier 2
  (the oracle) values and bounds for brier / ignorance / rps:
  dict name -> (tier-1 ref, tier-1 bound, oracle, tier-2 bound), plus the
  saturation band mask."""
  thr = case.thresholds()
  mean, std, t = case.mean, case.std, case.t
  lo, hi = tc.bracket(thr)
  with np.errstate(all='ignore'):
    t_gt = t[None] > lo
    t_lt = t[None] < hi
    zn = tc.emulate_z(thr, mean[None], std[None])
    upside = zn > 0
    a32, tail32 = tc.emulate_tail(zn)
    a64 = np.abs(zn).astype(F64) * 0.70710678118654752
    tail64 = 0.5 * special.erfc(a64)
    far = tail32 < tc.TAIL_SWITCH
    # where the float32 tail is within erfcf's error of the switch the kernel
    # may take either branch: tier 1 is skipped there (tier 2 still holds)
    ambiguous = np.abs(tail32 - tc.TAIL_SWITCH) <= 8 * U * tc.TAIL_SWITCH
    tail_e = np.where(far, tail64, tail32)
    # tier 1: erfcf is within 4 ulp (8u relative) of erfc(a) in float32; the
    # float64 erfc within 5 ulp, and its argument a64 one rounding (2^-53)
    # off the float64 product the emulation forms
    rel1 = np.where(far, (tc.ULP_ERFC64 + 2) * 2.0 ** -52,
                    tc.ULP_ERFCF * 2 * U)
    ref1 = tc.reference_scores(tail_e, upside, t_gt, t_lt)
    b1 = tc.score_bounds(tail_e, rel1, upside, t_gt, t_lt, *ref1)
    # tier 2: z itself is off by three float32 roundings (difference,
    # reciprocal, product); a by one more and by the float32 constant
    # 0.70710678f (D_C relative) on the float32 path, so the tail is off by
    # rel_tail_from_a(a, delta_a) ~ z^2 * delta_a on top of tier 1
    mean64, std64 = mean.astype(F64)[None], std.astype(F64)[None]
    z64 = (thr - mean64) / std64
    a_true = np.abs(z64) / np.sqrt(2.0)
    tail_true = 0.5 * special.erfc(a_true)
    delta_a = np.where(far, 3 * U + 2.0 ** -52, 4 * U + tc.D_C)
    rel2 = rel1 + tc.rel_tail_from_a(a_true, delta_a)
    want = case.oracle(False)
    orc = (want[..., 0], want[..., 2], want[..., 3])
    b2 = tc.score_bounds(tail_true, rel2, upside, t_gt, t_lt, *orc)
    # the ignorance saturates where 1 - tail rounds to 1 (tail <= 2^-54);
    # kernel and reference may disagree only where their tails straddle it
    band = np.abs(tail_true - tc.SATURATION) <= rel2 * tail_true
    # and the reference's erfc (scipy) is 0 past a^2 = 709.78 (|z| > 37.68),
    # where the kernel follows it: again only the z rounding can straddle it
    band |= np.abs(a_true ** 2 / tc.ERFC_UNDERFLOW - 1) <= 2 * delta_a
  fix = lambda b: np.nan_to_num(b, nan=0.0, posinf=np.inf)
  names = ('brier', 'ignorance', 'rps')
  return ({n: (ref1[i], fix(b1[i]), orc[i], fix(b2[i]))
           for i, n in enumerate(names)}, band, ambiguous, tail_true)


@pytest.mark.parametrize('case', [c for c in tc.gaussian_cases() if c.nq],
                         ids=lambda c: c.name)
def test_gaussian_threshold_scores_in_two_tiers(ctx, case):
  got = gauss_point(ctx, case)
  refs, band, ambiguous, tail_true = gauss_reference(case)
  # the saturation band is narrow, and cells sit just outside it both ways
  near = np.abs(tail_true / tc.SATURATION - 1)
  assert band.sum() <= 4 * case.nq
  if case.nq == 1:  # the cells of gaussian_z_grid() straddle it
    assert ((near < 0.02) & ~band & (tail_true < tc.SATURATION)).any()
    assert ((near < 0.02) & ~band & (tail_true > tc.SATURATION)).any()
  for k, name in ((0, 'brier'), (2, 'ignorance'), (3, 'rps')):
    g = got[..., k]
    ref1, b1, orc, b2 = refs[name]
    keep = ~band
    assert_same_specials(np.where(keep, g, 0), np.where(keep, orc, 0),
                         f'{case.name} {name}')
    t1 = keep & ~ambiguous
    assert_within(np.where(t1, g, 0), np.where(t1, ref1, 0), b1,
                  f'{case.name} {name} tier 1')
    assert_within(np.where(keep, g, 0), np.where(keep, orc, 0), b2,
                  f'{case.name} {name} tier 2')
  np.testing.assert_array_equal(got[..., 1], 0.0)


def test_gaussian_crps_and_variance(ctx):
  case = [c for c in tc.gaussian_cases() if c.nq == 0][0]
  got = gauss_point(ctx, case)[0]
  want = case.oracle(False)[0]
  mean, std, t = case.mean, case.std, case.t
  with np.errstate(all='ignore'):
    zn = ((mean - t).astype(F32) / std).astype(F32)
    az = np.abs(zn).astype(F64)
    a = (np.abs(zn) * F32(tc.C_SQRT1_2)).astype(F32).astype(F64)
    tail = special.erfc(a)
    pdf = np.exp(-0.5 * az * az) / np.sqrt(2 * np.pi)
    s = std.astype(F64)
    ref1 = s * (az * (1 - tail) + 2 * pdf - 1 / np.sqrt(np.pi))
    # bracket az (1 - tail) + 2 pdf - 1/sqrt(pi): erfcf 4 ulp on the tail,
    # one rounding of 1 - tail and of the product; expf 2 ulp, the float32
    # -0.5 zn zn (two roundings: u z^2 in the exponent), the float32
    # constants 0.39894228f / 0.56418958f and a product; two sums; times std
    c_pdf = abs(float(F32(0.39894228)) * np.sqrt(2 * np.pi) - 1)
    c_pi = abs(float(F32(0.56418958)) * np.sqrt(np.pi) - 1)
    A, B, C = az * (1 - tail), 2 * pdf, 1 / np.sqrt(np.pi)
    e1 = (az * (8 * U * tail + 2 * U) + B * (4 * U + U * az * az + c_pdf + U)
          + C * c_pi + 2 * U * (A + B + C))
    b1 = np.nan_to_num(s * e1 + U * np.abs(ref1), nan=0.0, posinf=np.inf)
    # tier 2: zn is off by two roundings (mean - t, the quotient): d crps / dz
    # = std (2 Phi(z) - 1), |.| <= std; and a by one more plus D_C
    e2 = az * 2 * U + az * tail * tc.rel_tail_from_a(a, U + tc.D_C)
    b2 = np.nan_to_num(b1 + s * e2 + U * np.abs(want[:, 0]), nan=0.0,
                       posinf=np.inf)
  assert_same_specials(got[:, 0], want[:, 0], 'crps')
  assert_within(got[:, 0], ref1, b1, 'crps tier 1')
  assert_within(got[:, 0], want[:, 0], b2, 'crps tier 2')
  np.testing.assert_array_equal(got[:, 1], (std * std).astype(F64))
  assert_same_specials(got[:, 1], want[:, 1], 'variance')


# -- reductions ---------------------------------------------------------------------
def _weights(r, cell_w_addr, zero_skip):
  from weatherbench2_b200 import _lib
  return _lib.WeightSpec(cell_w_dev=cell_w_addr, zero_skip=zero_skip,
                         **r['weights'])


def _run_reduction(c, r, kind, form, zero_skip, skipna, dev, fields=None):
  """Calls the entry on context `c` (real or FakeContext) with arrays on the
  device (`dev`) or in host memory; returns [nfield][nq][nregion][8]."""
  import torch
  nf = r['nfield'] if fields is None else fields
  cells = r['cells']
  keep = []  # the arrays behind the addresses live until the call returns

  def put(a):
    a = np.ascontiguousarray(a)
    if dev:
      d = _dev(a)
      keep.append(d)
      return d.data_ptr()
    keep.append(a)
    return a.ctypes.data

  def rep(a):  # the case's fields, repeated up to nf fields
    return np.concatenate([a] * (nf // a.shape[-3]), axis=-3)

  cell_w = put(r['cell_w'])
  w = _weights(r, cell_w, zero_skip)
  off = np.arange(nf, dtype=np.int64) * cells
  nq = 0 if kind == 'crps' else (4 if form == 'field' else 3)
  z = np.array([-1.2, 0.3, 0.9]) if form == 'gauss' else None
  if form == 'field':
    thr = rep(r['thr'])
    a, offa, b, offb = put(thr), (np.arange(nq)[:, None] * nf * cells +
                                  off[None]).reshape(-1), None, None
  elif form == 'gauss':
    a, offa, b, offb = put(rep(r['cm'])), off, put(rep(r['cs'])), off
  else:
    a = offa = b = offb = None
  res = np.full((nf, max(nq, 1), w.nregion, 8), 7.0)
  if dev:
    out_t = torch.from_numpy(res).cuda()
    out = out_t.data_ptr()
  else:
    out = res.ctypes.data
  if kind == 'ens':
    x = rep(r['x'])
    c.ens_threshold_metrics(put(x), put(rep(r['t'])), r['m'], nf * cells, off,
                            off, nq, a, offa, b, offb, z, w, skipna, out)
  else:
    c.gaussian_metrics(put(rep(r['mean'])), put(rep(r['std'])),
                       put(rep(r['t'])), off, off, off, nq, a, offa, b, offb,
                       z, w, skipna, out)
  return out_t.cpu().numpy() if dev else res


REDUCTIONS = [('ens', 'gauss'), ('ens', 'field'), ('gauss', 'gauss'),
              ('gauss', 'field'), ('crps', None)]


@pytest.mark.parametrize('skipna', [False, True])
@pytest.mark.parametrize('zero_skip', [False, True])
@pytest.mark.parametrize('kind,form', REDUCTIONS)
def test_weighted_sums_match_the_interpretation(ctx, kind, form, zero_skip,
                                                skipna):
  """Sums of float32 point values over regions, longitude boxes, column and
  cell weights: about 1e-6 relative to the interpretation.  NaN in
  zero-weight cells poisons nothing with zero_skip and everything without
  it (unless skipna)."""
  import fake_ctx
  r = tc.reduction_case()
  got = _run_reduction(ctx, r, kind, form, zero_skip, skipna, True)
  want = _run_reduction(fake_ctx.FakeContext(), r, kind, form, zero_skip,
                        skipna, False)
  # the slots the header defines: all eight for the ensemble; brier,
  # ignorance, rps part and their weight sums, or crps, std^2 and theirs
  slots = {'ens': list(range(8)), 'gauss': [0, 2, 3, 4, 6, 7],
           'crps': [0, 1, 4, 5]}[kind]
  got, want = got[..., slots], want[..., slots]
  assert_same_specials(got, want, f'{kind} {form}')
  np.testing.assert_allclose(got, want, rtol=1e-6, atol=1e-9)
  poisoned = np.isnan(got[..., 0]).all()
  if kind == 'ens':  # NaN members sit in weighted cells too
    assert poisoned == (not skipna)
  else:
    assert poisoned == (not zero_skip and not skipna)
    assert not np.isnan(got[..., 0]).any() or poisoned


@pytest.mark.parametrize('kind,form', [('ens', 'gauss'), ('gauss', 'gauss'),
                                       ('crps', None)])
def test_a_field_alone_matches_the_same_field_in_a_large_launch(ctx, kind, form):
  """One field runs in 4-row blocks, 300 fields in 8-row blocks."""
  r = tc.reduction_case(nfield=1)
  one = _run_reduction(ctx, r, kind, form, True, True, True)
  many = _run_reduction(ctx, r, kind, form, True, True, True, fields=300)
  np.testing.assert_allclose(many[0], one[0], rtol=1e-13, atol=1e-300)
  np.testing.assert_allclose(many[-1], one[0], rtol=1e-13, atol=1e-300)


@pytest.mark.parametrize('skipna', [False, True])
def test_grouped_maps_average_over_valid_groups(ctx, skipna):
  """ngroup = 3 slabs per map, NaN members and truth: the time mean of the
  maps entry against the interpretation (skipna divides by the number of
  valid groups per cell)."""
  import torch
  import fake_ctx
  rs = np.random.RandomState(7)
  nout, ngroup, nrow, ncol, m, nq = 2, 3, 5, 70, 6, 3
  nf, cells = nout * ngroup, nrow * ncol
  x = rs.randint(-2, 3, size=(m, nf, cells)).astype(F32)
  x[rs.rand(*x.shape) < 0.3] = np.nan
  t = rs.randint(-2, 3, size=(nf, cells)).astype(F32)
  t[rs.rand(*t.shape) < 0.3] = np.nan
  thr = (rs.randint(-2, 3, size=(nq, nf, cells)) + 0.5).astype(F32)
  off = np.arange(nf, dtype=np.int64) * cells
  offa = (np.arange(nq)[:, None] * nf * cells + off[None]).reshape(-1)
  for stat in range(4):
    res = []
    for c in (ctx, fake_ctx.FakeContext()):
      if c is ctx:
        xs, ts, ths = _dev(x), _dev(t), _dev(thr)
        out = torch.full((nq, nout, nrow, ncol), 7.0, device='cuda')
        p = lambda a: a.data_ptr()
      else:
        xs, ts, ths = x, t, thr
        out = np.full((nq, nout, nrow, ncol), 7.0, F32)
        p = lambda a: a.ctypes.data
      c.ens_threshold_maps(p(xs), p(ts), m, nf * cells, nout, ngroup, off, off,
                           nq, p(ths), offa, None, None, None, nrow, ncol, ncol,
                           stat, skipna, p(out))
      res.append(out.cpu().numpy() if c is ctx else out)
    assert_same_specials(res[0], res[1], f'stat {stat}')
    np.testing.assert_allclose(res[0], res[1], rtol=1e-6, atol=1e-7)


# -- argument errors -----------------------------------------------------------------
def test_argument_errors_raise_and_launch_nothing(ctx):
  import ctypes as C
  import torch
  from weatherbench2_b200 import _lib
  n = 8
  x, t = _dev(np.zeros((2, n), F32)), _dev(np.zeros(n, F32))
  thr = _dev(np.zeros((2, n), F32))
  out = torch.zeros(4096 * 8 * n, dtype=torch.float64, device='cuda')
  outf = torch.zeros(4097 * n, device='cuda')
  c = np.arange(n, dtype=np.int64)
  g = tc.geometry_1x1()
  z = np.zeros(1)

  def ens(nq=1, m=2, b=None, offb=None, zz=None):
    offa = np.zeros(max(nq, 1) * n, np.int64)
    return lambda: ctx.ens_threshold_metrics(
        x.data_ptr(), t.data_ptr(), m, n, c, c, nq, thr.data_ptr(), offa, b,
        offb, zz, g, False, out.data_ptr())

  def maps(nq=1, m=2, stat=0, nrow=1, ncol=n, stride=n, b=None, offb=None,
           zz=None):
    offa = np.zeros(max(nq, 1), np.int64)
    return lambda: ctx.ens_threshold_maps(
        x.data_ptr(), t.data_ptr(), m, n, 1, 1, c[:1], c[:1], nq,
        thr.data_ptr(), offa, b, offb, zz, nrow, ncol, stride, stat, False,
        outf.data_ptr())

  def gauss(nq=1, b=None, offb=None, zz=None):
    return lambda: ctx.gaussian_metrics(
        x.data_ptr(), x.data_ptr(), t.data_ptr(), c, c, c, nq, thr.data_ptr(),
        c, b, offb, zz, g, False, out.data_ptr())

  w = g.as_struct()
  cases = [
      ('nthreshold must be >= 1', ens(nq=0)),
      ('nthreshold out of range', ens(nq=4097)),
      ('nthreshold out of range', maps(nq=4097)),
      ('nthreshold out of range', maps(nq=0)),
      ('nthreshold out of range', gauss(nq=4097)),
      ('nmember out of range', ens(m=0)),
      ('nmember out of range', ens(m=65537)),
      ('nmember out of range', maps(m=0)),
      ('nmember out of range', maps(m=65537)),
      ('stat must be 0..3', maps(stat=4)),
      ('need off_b and z', ens(b=thr.data_ptr(), offb=c)),
      ('need off_b and z', ens(b=thr.data_ptr(), zz=z)),
      ('need off_b and z', maps(b=thr.data_ptr(), offb=c[:1])),
      ('need off_b and z', maps(b=thr.data_ptr(), zz=z)),
      ('need off_b and z', gauss(b=thr.data_ptr(), offb=c)),
      ('need off_b and z', gauss(b=thr.data_ptr(), zz=z)),
      ('bad grid', maps(nrow=0)),
      ('bad grid', maps(stride=n - 1)),
      ('only WB2_F32', lambda: _lib.check(ctx.lib.wb2_ens_threshold_metrics(
          ctx.handle, C.c_void_p(x.data_ptr()), C.c_void_p(t.data_ptr()),
          _lib.F64, 2, n, n, c.ctypes.data_as(C.POINTER(C.c_int64)),
          c.ctypes.data_as(C.POINTER(C.c_int64)), 1,
          C.c_void_p(thr.data_ptr()), c.ctypes.data_as(C.POINTER(C.c_int64)),
          None, None, None, C.byref(w), 0, C.c_void_p(out.data_ptr())))),
      ('only WB2_F32', lambda: _lib.check(ctx.lib.wb2_ens_threshold_maps(
          ctx.handle, C.c_void_p(x.data_ptr()), C.c_void_p(t.data_ptr()),
          _lib.F64, 2, n, 1, 1, c.ctypes.data_as(C.POINTER(C.c_int64)),
          c.ctypes.data_as(C.POINTER(C.c_int64)), 1,
          C.c_void_p(thr.data_ptr()), c.ctypes.data_as(C.POINTER(C.c_int64)),
          None, None, None, 1, n, n, 0, 0, C.c_void_p(outf.data_ptr())))),
      ('only WB2_F32', lambda: _lib.check(ctx.lib.wb2_gaussian_metrics(
          ctx.handle, C.c_void_p(x.data_ptr()), C.c_void_p(x.data_ptr()),
          C.c_void_p(t.data_ptr()), _lib.F64, n,
          c.ctypes.data_as(C.POINTER(C.c_int64)),
          c.ctypes.data_as(C.POINTER(C.c_int64)),
          c.ctypes.data_as(C.POINTER(C.c_int64)), 0, None, None, None, None,
          None, C.byref(w), 0, C.c_void_p(out.data_ptr())))),
  ]
  for msg, call in cases:
    before = ctx.launch_count
    with pytest.raises(_lib.Wb2Error, match=msg):
      call()
    assert ctx.launch_count == before, msg

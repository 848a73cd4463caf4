"""The cases of threshold_cases.py reach what they claim, the NumPy stand-in
(fake_ctx.py) interprets their raw arguments as the oracle does, and the
float32-z model of the Gaussian kernel agrees with the oracle within the
bounds test_threshold_abi_gpu.py holds the kernel to.  No GPU needed."""
import numpy as np
import pytest
from scipy import special

import fake_ctx
from oracle import wb2_oracle as orc
import threshold_cases as tc
from threshold_cases import F32, F64, U


def test_bracket_cases_sit_at_lo_and_hi():
  case, fma = tc.bracket_cases()
  thr = case.thresholds()
  lo, hi = tc.bracket(thr)
  k = np.arange(case.ncell) % case.nq
  c = np.arange(case.ncell)
  lo_c, hi_c = lo[k, c], hi[k, c]
  x = case.members
  assert (x == lo_c).sum() > 300 and (x == hi_c).sum() > 300
  assert (x == tc.down(lo_c)).sum() > 300 and (x == tc.up(hi_c)).sum() > 300
  exact = lo_c == hi_c  # thr is a float32 number (z = 0, std = 0)
  assert exact.sum() > 100 and (~exact).sum() > 300
  assert ((case.t == lo_c) & ~exact).sum() > 20
  assert ((case.t == hi_c) & ~exact).sum() > 20
  # beyond float32 range: lo = FLT_MAX, hi = inf and mirrored
  assert ((lo == np.finfo(F32).max) & np.isposinf(hi)).any()
  assert (np.isneginf(lo) & (hi == -np.finfo(F32).max)).any()
  assert np.isinf(x).any() and (x == np.finfo(F32).max).any()
  # fma: threshold k of cell k is a float32 x after two roundings only
  assert tc.fma_cells_in(fma) == 16
  # M = 8: the float32 emulation equals the oracle bit for bit
  for cs in (case, fma):
    want = cs.oracle(False)
    b32, r32, _ = tc.ens_emulate(cs, False)
    np.testing.assert_array_equal(b32.astype(F64), want[..., 0])
    np.testing.assert_array_equal(r32.astype(F64), want[..., 3])


def test_fma_cells_change_a_comparison():
  """With one rounding, the fma cells' members at x would count differently."""
  _, fma = tc.bracket_cases()
  diff = 0
  for c in range(16):
    one = tc.fma_single_rounding(fma.thr_a[c], fma.thr_b[c], fma.z[c])
    lo1, hi1 = tc.bracket(np.array([one]))
    x = fma.members[:, c]
    lo2, hi2 = tc.bracket(fma.thresholds()[c, c:c + 1])
    diff += ((x > lo1[0]) != (x > lo2[0])).sum() + ((x < hi1[0]) != (x < hi2[0])).sum()
    # and the scores move (the truth sits off x; with a symmetric placement
    # the changed counts could leave every score as it was)
    t64 = fma.t[c:c + 1].astype(F64)
    def scores(thr):
      th = np.array([thr])
      return (orc.ens_brier_pointwise(x.astype(F64)[:, None], t64, th, 0,
                                      False, False)[0],
              orc.ens_rps_part_pointwise(x.astype(F64)[:, None], t64, th, 0,
                                         False)[0])
    assert scores(one) != scores(float(fma.thresholds()[c, c]))
  assert diff >= 16


def test_warp_cases_take_each_path():
  case, kinds = tc.warp_cases()
  strict = tc.warp_strictness(case)
  assert case.nq == 5 and len(strict) == 2  # passes of 4 and 1
  for w, kind in enumerate(kinds):
    assert strict[0][w] == (kind != 'onelane'), (w, kind)
    assert not strict[1][w]


def test_member_count_cases_cover_nvalid_and_quotients():
  cases = tc.member_count_cases()
  ms = sorted({c.nmember for c in cases})
  assert ms == [1, 2, 24, 25, 26, 49, 51, 64, 65, 257, 5000]
  assert {c.interleaved for c in cases} == {False, True}
  newton_matters = False
  for c in cases:
    nvalid = (~np.isnan(c.members)).sum(0)
    assert nvalid[0] == 0 and nvalid[1] == 1 and (nvalid[2:6] == c.nmember).all()
    assert np.isnan(c.t).any() and np.isinf(c.t).any() and np.isinf(c.members).any()
    _, _, (c_gt, c_lt, nv) = tc.ens_emulate(c, True)
    for cnt in (c_gt, c_lt):
      for d in (nv[None], F32(c.nmember)):
        with np.errstate(all='ignore'):
          q = cnt / d
          naive = cnt * (F32(1) / d)
        newton_matters |= bool(((q != naive) & np.isfinite(q)).any())
  # a quotient c * (1 / n) without the Newton step differs somewhere
  assert newton_matters


def test_threshold_counts_cover_every_pass_mix():
  mixes = set()
  for c in tc.threshold_count_cases():
    left, mix = c.nq, []
    while left:
      tq = 4 if left >= 4 else 2 if left >= 2 else 1
      mix.append(tq)
      left -= tq
    mixes.add(tuple(mix))
  assert {(1,), (2,), (2, 1), (4,), (4, 1), (4, 2, 1), (4, 4, 1)} <= mixes


def test_field_cases_have_ties_and_nan_thresholds():
  (c,) = tc.field_cases()
  thr = c.thresholds()
  assert (c.members[None] == thr[:, None]).sum() > 500
  assert np.isnan(thr).sum() > 50


def test_gaussian_grid_reaches_every_band():
  z = tc.gaussian_z_grid()
  for v in (0, 1e-30, 0.5, 1, 3, 6, 8, 20, 40, np.inf):
    assert v in z and (v == 0 or -v in z)
  tail = 0.5 * special.erfc(np.abs(z[np.isfinite(z)]) / np.sqrt(2))
  assert ((tail > tc.TAIL_SWITCH) & (tail < 2 * tc.TAIL_SWITCH)).any()
  assert ((tail < tc.TAIL_SWITCH) & (tail > tc.TAIL_SWITCH / 2)).any()
  sat = np.abs(tail / tc.SATURATION - 1)
  assert ((sat < 0.02) & (tail < tc.SATURATION)).any()
  assert ((sat < 0.02) & (tail > tc.SATURATION)).any()
  cases = tc.gaussian_cases()
  g = cases[0]
  assert np.isnan(g.t).any() and np.isnan(g.std).any() and (g.std == 0).any()
  assert np.isinf(g.std).any() and np.isinf(g.mean).any() and np.isnan(g.mean).any()
  assert np.isnan(g.thresholds()).any()
  assert (np.abs(g.thresholds()) > np.finfo(F32).max).any()
  assert {c.nq for c in cases} == {0, 1, 7}


def _run_fake_point(case, skipna):
  """The stand-in on a case, one field per cell: [nq][ncell][8]."""
  from weatherbench2_b200 import _lib
  ctx = fake_ctx.FakeContext()
  n = case.ncell
  c = np.arange(n, dtype=np.int64)
  keep = []

  def put(a):
    a = np.ascontiguousarray(a)
    keep.append(a)
    return a.ctypes.data

  a, b = case.thr_buffers() if case.nq else (None, None)
  off_a, off_b = case.off_thr() if case.nq else (None, None)
  out = np.zeros((n, max(case.nq, 1), 1, 8))
  g = _lib.WeightSpec(1, 1, np.ones((1, 1)), [0, 1], np.ones((1, 1)))
  if case.kind == 'ens':
    ctx.ens_threshold_metrics(put(case.x_buffer()), put(case.t), case.nmember,
                              case.member_stride(), case.off_x(), c, case.nq,
                              put(a), off_a, None if b is None else put(b),
                              off_b, case.z, g, skipna, out.ctypes.data)
  else:
    ctx.gaussian_metrics(put(case.mean), put(case.std), put(case.t), c, c, c,
                         case.nq, None if a is None else put(a), off_a,
                         None if b is None else put(b), off_b, case.z, g,
                         skipna, out.ctypes.data)
  return out[:, :, 0].transpose(1, 0, 2)


@pytest.mark.parametrize('skipna', [False, True])
def test_fake_context_matches_the_oracle(skipna):
  cases = (tc.bracket_cases() + tc.field_cases() +
           [c for c in tc.member_count_cases() if c.nmember < 1000] +
           tc.threshold_count_cases()[:4] + tc.gaussian_cases())
  for case in cases:
    got = _run_fake_point(case, skipna)
    want = case.oracle(skipna)
    stats = (0, 1, 2, 3) if case.kind == 'ens' else (
        (0, 1) if case.nq == 0 else (0, 2, 3))
    for k in stats:
      w = got[..., 4 + k]
      v = np.where(w == 0, np.nan, got[..., k])
      # NumPy's pairwise sums differ in the last bit between a 1-cell
      # slab and the whole case
      np.testing.assert_allclose(v, want[..., k], rtol=1e-14, atol=1e-15,
                                 err_msg=f'{case.name} {k}')


def test_float32_z_model_agrees_with_the_oracle():
  """The float32-z emulation's tail is within the tier-2 bound of the exact
  tail, away from zero / infinite / NaN z."""
  for case in tc.gaussian_cases():
    if not case.nq:
      continue
    thr = case.thresholds()
    with np.errstate(all='ignore'):
      zn = tc.emulate_z(thr, case.mean[None], case.std[None])
      a32, tail32 = tc.emulate_tail(zn)
      z64 = (thr - case.mean.astype(F64)[None]) / case.std.astype(F64)[None]
      a = np.abs(z64) / np.sqrt(2)
      tail = 0.5 * special.erfc(a)
      ok = np.isfinite(z64) & (tail > 1e-300) & (tail32 >= tc.TAIL_SWITCH)
      rel = np.abs(tail32[ok] / tail[ok] - 1)
      bound = tc.rel_tail_from_a(a[ok], 4 * U + tc.D_C)
    assert ok.sum() > 50
    assert (rel <= bound).all()
    # and the bound is not vacuous: well below 1e-3 relative everywhere here
    assert bound.max() < 1e-3
    assert (np.sign(zn[ok]) == np.sign(z64[ok])).all()

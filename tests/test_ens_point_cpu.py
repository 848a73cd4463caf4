"""The point cases of ens_point_cases.py without a GPU: they reach the paths
they claim, their float64 reference is the oracle's, and float32 models of
the kernels' spread arithmetic show that the bounds can see the error of a
rank sum formed on raw members (the raw model fails them at realistic
magnitudes) while the mean-removed sums of every path pass them."""
import numpy as np
import pytest

import ens_point_cases as epc
from ens_point_cases import U
from test_kernel_arithmetic_models import NETS, _expand

F = np.float32
CASES = epc.cases()


def test_member_counts_reach_every_bucket_and_path():
  for mp in (2, 3, 4, 5, 8, 10, 16, 20, 32, 50, 64):
    assert mp in epc.MEMBER_COUNTS  # exact
    if mp not in (3, 4, 5):         # 3, 4 and 5 have no padded member count
      assert any(epc.bucket(m) == (mp, False) for m in epc.MEMBER_COUNTS)
  assert 64 in epc.MEMBER_COUNTS and 65 in epc.MEMBER_COUNTS
  want = {
      (8, False, (), 'pair'): 'pair', (8, False, ('s',), 'pair'): 'twin',
      (8, False, ('s', 'e'), 'pair'): 'scalar', (8, True, (), 'pair'): 'scalar',
      (8, False, (), 'odd'): 'twin', (51, False, (), 'pair'): 'scalar',
      (5, False, (), 'pair'): 'scalar', (1, False, (), 'pair'): 'scalar',
      (65, False, (), 'pair'): 'big', (1551, True, (), 'pair'): 'big',
  }
  for (M, sk, e, lay), path in want.items():
    env = {}
    if 's' in e:
      env['WB2_ENS_PATH'] = 'scalar'
    if 'e' in e:
      env['WB2_ENS_SORT'] = 'exact'
    assert epc.metrics_path(M, sk, env, lay) == path, (M, sk, env, lay)
  assert epc.maps_path(50, False) == 'twin' and epc.maps_path(51, False) == 'scalar'
  assert epc.maps_path(50, True) == 'scalar'


@pytest.mark.parametrize('M', [1, 2, 5, 51, 100])
def test_nan_and_inf_patterns(M):
  case = CASES[M]
  for skipna in (False, True):
    ref = epc.reference(case, skipna)
    for lab, stat, want in (('nan1', 'spread', None if skipna or M == 1 else 'nan'),
                            ('nanall', 'skill', 'nan'), ('nant', 'mse', 'nan'),
                            ('nant', 'spread', 'finite'), ('pinf', 'skill', 'inf'),
                            ('pinf', 'var', 'nan'),
                            ('tninf', 'mse', 'inf'), ('tpinf', 'var', 'finite' if M > 1 else 'nan')):
      v = ref[stat][case.mask(lab)]
      if want == 'nan':
        assert np.isnan(v).all(), (lab, stat, skipna)
      elif want == 'inf':
        assert (v == np.inf).all(), (lab, stat, skipna)
      elif want == 'finite':
        assert np.isfinite(v).all(), (lab, stat, skipna)
    if skipna and M > 1:
      assert np.isfinite(ref['spread'][case.mask('nan1')]).all()
      assert np.isnan(ref['var'][case.mask('nanall_but1')]).all()
      # one valid member: the coefficient keeps M, the spread is -2 x
      x = np.nansum(case.x[:, case.mask('nanall_but1')].astype(np.float64), axis=0)
      np.testing.assert_allclose(ref['spread'][case.mask('nanall_but1')], -2 * x)


@pytest.mark.parametrize('M', epc.MEMBER_COUNTS)
def test_reference_is_the_oracles(M):
  from oracle import wb2_oracle as orc
  case = CASES[M]
  dims = ('realization', 'cell')
  for skipna in (False, True):
    ref = epc.reference(case, skipna)
    sp, _ = orc.pointwise_crps_spread(case.x, dims, 'realization', skipna)
    np.testing.assert_array_equal(ref['spread'], sp)
    bnd = epc.bounds(case, skipna, 'scalar', ref)
    sk, _ = orc.pointwise_crps_skill(case.x, dims, case.t, ('cell',),
                                     'realization', skipna)
    ok = np.isfinite(ref['skill'])
    with np.errstate(invalid='ignore'):
      assert (np.abs(sk - ref['skill'])[ok] <= bnd['skill'][ok]).all()
    np.testing.assert_array_equal(np.isnan(sk), np.isnan(ref['skill']))
  fin = case.finite()
  bf = epc.brute_force_spread(case) if M <= 100 else None
  if bf is not None:
    ref = epc.reference(case, False)['spread']
    np.testing.assert_allclose(ref[fin], bf[fin], rtol=1e-12,
                               atol=1e-9 * np.abs(case.x[:, fin]).max())


def test_equal_values_have_exact_float32_means():
  for c in epc.EQUAL_VALUES:
    for M in epc.MEMBER_COUNTS:
      s = F(0)
      for _ in range(M):
        s = F(s + F(c))
      assert F(s / F(M)) == F(c), (c, M)  # skipna and K2b: division
      if M <= 64:  # the reciprocal of launch_ens / ens_pair_kernel
        assert F(s * F(1.0 / M)) == F(c), (c, M)


# ---- float32 models of the spread arithmetic -----------------------------------------
def _fma_chain(coef, v):
  """s = fma(c_i, v_i, s) over i, one float32 rounding per step."""
  s = np.zeros(v.shape[1], np.float32)
  for i in range(v.shape[0]):
    s = (s.astype(np.float64) + np.float64(coef[i]) * v[i].astype(np.float64)).astype(F)
  return s


def _network(v, mp, kind, phase=0):
  """Replays SortNet<mp> / SortNetTwin<mp>: 'minmax' exact, 'twin' the
  (a + b) - lo form on every CE2 comparator, 'pair' on two of three."""
  v = v.copy()
  if kind == 'twin':
    ops = []
    for op, a, b in NETS[('SortNetTwin', mp)]:
      ops += [(op, a, b)] + ([(op, a + 1, b + 1)] if op == 'CE2' else [])
  else:
    ops = [('CE', a, b) for a, b in _expand(NETS[('SortNet', mp)])]
  for k, (op, a, b) in enumerate(ops):
    lo = np.minimum(v[a], v[b])
    inexact = (kind == 'twin' and op == 'CE2') or (kind == 'pair' and (k + phase) % 3)
    hi = (v[a] + v[b]) - lo if inexact else np.maximum(v[a], v[b])
    v[a], v[b] = lo, hi
  return v


def model_spread(x, kind, phase=0):
  """float32 spread of the finite points x [M][n] on one path's arithmetic:
  'raw' the rank sum on the sorted raw members (the parent's scalar network
  and K2b order), 'scalar' / 'twin' / 'pair' on the mean-removed members."""
  M = x.shape[0]
  s = np.zeros(x.shape[1], np.float32)
  for m in range(M):
    s = F(s + x[m])
  mean = F(s * F(1.0 / M))
  coef = (2 * np.arange(1, M + 1) - M - 1).astype(F)
  if kind == 'raw':
    v = np.sort(x, axis=0)
  else:
    v = (x - mean).astype(F)
    v = np.sort(v, axis=0) if kind == 'scalar' else _network(v, M, kind, phase)
  s = _fma_chain(coef, v)
  return F(F(2) * F(s * F(1.0 / M)) * F(1.0 / (M - 1)))


MAG_M = [5, 7, 8, 16, 50, 51, 64]


@pytest.mark.parametrize('M', MAG_M)
def test_raw_rank_sum_fails_the_spread_bound_and_mean_removed_sums_pass(M):
  case = CASES[M]
  mag = case.mask('mag') & case.finite()
  x = case.x[:, mag]
  ref = epc.reference(case, False)['spread'][mag]
  mu = np.array([float(l.split(':')[1]) for l in np.array(case.labels)[mag]])
  ratio = np.array([float(l.split(':')[2]) for l in np.array(case.labels)[mag]])
  kinds = ['scalar'] + (['twin', 'pair'] if M in (8, 16, 50, 64) else [])
  for kind in kinds:
    path = 'scalar' if kind == 'scalar' else kind
    bnd = epc.bounds(case, False, path)['spread'][mag]
    for phase in ((0, 1, 2) if kind == 'pair' else (0,)):
      err = np.abs(model_spread(x, kind, phase).astype(np.float64) - ref)
      assert (err <= bnd).all(), (kind, phase, (err / bnd).max())
  raw = np.abs(model_spread(x, 'raw').astype(np.float64) - ref)
  bnd = epc.bounds(case, False, 'scalar')['spread'][mag]
  big = (np.abs(mu) >= 5e4) & (ratio <= 1e-3)
  assert (raw[big] > bnd[big]).any(), (raw / bnd).max()
  # the raw error scales with |x|, not with the spread: about 1e-4 of it here
  assert (raw / np.abs(ref))[big].max() > 2e-5


def test_raw_rank_sum_fails_the_bound_on_k2b_order():
  """K2b's per-lane partials and butterfly, on raw members (the parent) and
  on mean-removed members."""
  case = CASES[100]
  mag = case.mask('mag') & case.finite()
  x = case.x[:, mag]
  M = x.shape[0]
  ref = epc.reference(case, False)['spread'][mag]
  bnd = epc.bounds(case, False, 'big')['spread'][mag]
  rank = np.argsort(np.argsort(x, axis=0, kind='stable'), axis=0) + 1
  coef = (2 * rank - M - 1).astype(F)

  def k2b(v):
    lanes = np.zeros((32, v.shape[1]), np.float32)
    for m in range(M):
      lanes[m % 32] = (lanes[m % 32].astype(np.float64) +
                       coef[m].astype(np.float64) * v[m].astype(np.float64)).astype(F)
    for off in (16, 8, 4, 2, 1):
      lanes = F(lanes + lanes[np.arange(32) ^ off])
    s = lanes[0]
    return F(F(F(2) * F(s / F(M))) / F(M - 1)).astype(np.float64)

  s = np.zeros(x.shape[1], np.float32)
  for m in range(M):
    s = F(s + x[m])
  mean = F(s / F(M))
  assert (np.abs(k2b(x) - ref) > bnd).any()
  assert (np.abs(k2b(F(x - mean)) - ref) <= bnd).all()


def test_bound_is_scaled_by_dispersion_not_magnitude():
  case = CASES[51]
  b = epc.bounds(case, False, 'scalar')['spread']
  lab = np.array(case.labels)
  small = b[lab == 'mag:50000:0.0001:in'].max()
  assert small < 1e-4 * 5 * 51  # (M + 4) u times the dispersion, not 5e4
  assert small / U < 5e4

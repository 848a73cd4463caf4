"""The ensemble point statistics of K2 (wb2_ens_metrics: ens_pair_kernel, the
twin and scalar ens_metrics_kernel, K2b ens_big_kernel) and K6e
(wb2_ens_maps) called through `_lib.Context` directly, point by point, on the
seeded cases of ens_point_cases.py, against float64 references.

Reached here and nowhere else: members of mean 0 to 1e5 with spreads from
1e-4 to 1 of the mean, every dispatch bucket exact and padded on both sides of
the K2 / K2b switch (M = 1 to 1551), all-equal and +-0 ensembles, ties, a lone
outlier 1e6 spreads away, missing and infinite members and truth, with and
without skipna, on every path (forced with WB2_ENS_PATH / WB2_ENS_SORT, odd
offsets, skipna, M > 64).

Bounds are per point and per statistic, derived from the kernels' operation
order (ens_point_cases.bounds; DESIGN.md, K2): skill (M + 4) u skill; spread
(M + 4) u times the dispersion-weighted rank sum, plus 4 u (D + delta) per
comparator level on the (a + b) - lo networks and a mean|x| |n - M| term
under skipna with missing members; mse and var from the float32 mean's error
delta <= (n + 1) u mean|x_m|; debiased MSE the sum.  No global rtol.
Structural cases are exact (spread == var == 0 on all-equal members), and the
NaN / +inf / -inf pattern of every statistic equals the oracle's, except the
spread of an ensemble with an infinite member on the (a + b) - lo networks,
where inf - inf makes NaN (asserted non-finite).  M = 1: the kernels' variance
is 0 / 0 = NaN, as the reference's var(ddof=1); the operators replace it with
the reference's 0, as oracle.ensemble_variance does."""
import numpy as np
import pytest

import ens_point_cases as epc
from ens_point_cases import STATS, U

pytestmark = pytest.mark.gpu

CASES = {}


def _case(M):
  if M not in CASES:
    CASES[M] = epc.point_case(M)
  return CASES[M]


@pytest.fixture(scope='module')
def ctx():
  from weatherbench2_b200 import _lib
  return _lib.default_context(0)


def _dev(a):
  import torch
  return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _geometry():
  from weatherbench2_b200 import _lib
  return _lib.WeightSpec(1, 2, np.ones((1, 1)), [0, 2], np.ones((1, 1)))


def run_metrics(ctx, case, skipna, layout='pair', host=False):
  """[n / 2][10] float64 of wb2_ens_metrics: field f = points 2f, 2f + 1 on a
  1 x 2 geometry.  layout 'odd' shifts every offset by one element."""
  from weatherbench2_b200 import _lib
  import torch
  n, M = case.n, case.M
  shift = 1 if layout == 'odd' else 0
  x = np.concatenate([np.full(shift, np.nan, np.float32), case.x.ravel()])
  t = np.concatenate([np.full(shift, np.nan, np.float32), case.t])
  off = (shift + 2 * np.arange(n // 2)).astype(np.int64)
  if host:
    out = np.full((n // 2, 10), 7.0)
    ctx.ens_metrics_host(x.ctypes.data, t.ctypes.data, M, n, off, off,
                         _geometry(), skipna, out.ctypes.data)
    ctx.synchronize()
    return out
  xd, td = _dev(x), _dev(t)
  out = torch.full((n // 2, 10), 7.0, dtype=torch.float64, device='cuda')
  ctx.ens_metrics(xd.data_ptr(), td.data_ptr(), _lib.F32, M, n, off, off,
                  _geometry(), skipna, out.data_ptr())
  return out.cpu().numpy()


def run_maps(ctx, case, skipna):
  """[6][n] float32 of wb2_ens_maps (all six maps, ngroup = 1, one row)."""
  from weatherbench2_b200 import _lib
  import torch
  n = case.n
  xd, td = _dev(case.x), _dev(case.t)
  out = torch.full((6, 1, 1, n), 7.0, device='cuda')
  z = np.zeros(1, np.int64)
  ctx.ens_maps(xd.data_ptr(), td.data_ptr(), _lib.F32, case.M, n, 1, 1, z, z,
               1, n, n, 63, skipna, out.data_ptr())
  return out.cpu().numpy()[:, 0, 0]


def _pattern(a):
  return np.where(np.isnan(a), 0, np.where(a == np.inf, 1, np.where(a == -np.inf, 2, 3)))


def compare(got, ref, bnd, *, labels, M, path, env, exact=None, network=False):
  """Failures of got vs ref (name -> [k]) as printable lines."""
  bad = []
  for name in got:
    g, r, b = got[name], ref[name], bnd[name]
    fin = np.isfinite(r)
    with np.errstate(invalid='ignore', divide='ignore'):
      err = np.abs(g.astype(np.float64) - r)
      over = fin & ~(err <= b)
    pat = ~fin & (_pattern(g) != _pattern(r))
    if network and name in ('spread', 'crps'):
      # inf - inf of the (a + b) - lo comparators: NaN where the oracle has inf
      pat &= ~(np.isinf(r) & ~np.isfinite(g))
    if exact and name in exact:
      m, v = exact[name]
      over |= m & (g != v)
    for i in np.flatnonzero(over | pat):
      bad.append(f'M={M} path={path} env={env} point={i} ({labels[i]}) '
                 f'{name}: got {g[i]!r} want {r[i]!r} bound {b[i]:.3g} '
                 f'err/bound {err[i] / b[i] if b[i] else np.inf:.3g}')
  return bad


def _report(bad):
  assert not bad, f'{len(bad)} failures:\n' + '\n'.join(bad[:25])


def _pair_ref(ref, bnd, skipna, exact):
  """Mean of the two points of every field, its bound and count."""
  r2, b2, c2 = {}, {}, {}
  for k in ref:
    r = ref[k].reshape(-1, 2)
    b = bnd[k].reshape(-1, 2)
    ok = ~np.isnan(r) if skipna else np.ones_like(r, bool)
    cnt = ok.sum(axis=1).astype(np.float64)
    with np.errstate(invalid='ignore', divide='ignore'):
      r2[k] = np.where(ok, r, 0).sum(axis=1) / cnt if skipna else r.mean(axis=1)
      b2[k] = (np.where(ok, b + U * np.abs(r), 0).sum(axis=1) / cnt if skipna
               else (b + U * np.abs(r)).sum(axis=1) / 2)
    c2[k] = cnt
  ex = None
  if exact:
    ex = {k: (m.reshape(-1, 2).all(axis=1), v) for k, (m, v) in exact.items()}
  return r2, b2, c2, ex


VARIANTS = {
    # name: (env, skipna, layout)
    'default': ({}, False, 'pair'),
    'scalar': ({'WB2_ENS_PATH': 'scalar'}, False, 'pair'),
    'exact_sort': ({'WB2_ENS_PATH': 'scalar', 'WB2_ENS_SORT': 'exact'}, False,
                   'pair'),
    'skipna': ({}, True, 'pair'),
    'odd_offset': ({}, False, 'odd'),
}


def _setenv(monkeypatch, env):
  for k in ('WB2_ENS_PATH', 'WB2_ENS_SORT'):
    monkeypatch.delenv(k, raising=False)
  for k, v in env.items():
    monkeypatch.setenv(k, v)


@pytest.mark.parametrize('variant', list(VARIANTS))
@pytest.mark.parametrize('M', epc.MEMBER_COUNTS)
def test_ens_metrics_points(ctx, monkeypatch, M, variant):
  env, skipna, layout = VARIANTS[variant]
  case = _case(M)
  path = epc.metrics_path(M, skipna, env, layout)
  _setenv(monkeypatch, env)
  out = run_metrics(ctx, case, skipna, layout)
  ref = epc.reference(case, skipna)
  bnd = epc.bounds(case, skipna, path, ref)
  r2, b2, c2, ex = _pair_ref(ref, bnd, skipna,
                             epc.exact_expectations(case, skipna))
  labels = case.labels[::2]
  with np.errstate(invalid='ignore', divide='ignore'):
    got = {k: out[:, i] / out[:, 5 + i] for i, k in enumerate(STATS)}
  bad = compare(got, r2, b2, labels=labels, M=M, path=path, env=env, exact=ex,
                network=path in epc.NETWORK_PATHS)
  for i, k in enumerate(STATS):
    want = c2[k] if skipna else np.full(len(labels), 2.0)
    for j in np.flatnonzero(out[:, 5 + i] != want):
      bad.append(f'M={M} path={path} field={j} ({labels[j]}) {k} count '
                 f'{out[j, 5 + i]} want {want[j]}')
  _report(bad)


@pytest.mark.parametrize('skipna', [False, True])
@pytest.mark.parametrize('M', [m for m in epc.MEMBER_COUNTS if m <= 64])
def test_ens_maps_points(ctx, M, skipna):
  case = _case(M)
  path = epc.maps_path(M, skipna)
  maps = run_maps(ctx, case, skipna)
  ref = epc.reference(case, skipna)
  bnd = epc.bounds(case, skipna, path, ref)
  ref['crps'] = ref['skill'] - 0.5 * ref['spread']
  bnd['crps'] = bnd['skill'] + 0.5 * bnd['spread'] + 2 * U * np.abs(ref['crps'])
  got = dict(zip(STATS + ('crps',), maps))
  bad = compare(got, ref, bnd, labels=case.labels, M=M, path=f'maps_{path}',
                env={'skipna': skipna}, exact=epc.exact_expectations(case, skipna),
                network=path in epc.NETWORK_PATHS)
  _report(bad)


def _bits(a):
  return np.ascontiguousarray(a).view(np.uint64 if a.dtype == np.float64 else np.uint32)


@pytest.mark.parametrize('M,variant', [(50, 'default'), (50, 'scalar'),
                                       (50, 'exact_sort'), (51, 'default'),
                                       (16, 'skipna'), (100, 'default'),
                                       (100, 'skipna')])
def test_host_entry_gives_the_device_entry_bits(ctx, monkeypatch, M, variant):
  env, skipna, layout = VARIANTS[variant]
  case = _case(M)
  _setenv(monkeypatch, env)
  dev = run_metrics(ctx, case, skipna, layout)
  host = run_metrics(ctx, case, skipna, layout, host=True)
  np.testing.assert_array_equal(_bits(host), _bits(dev))


@pytest.mark.parametrize('M', [m for m in epc.MEMBER_COUNTS
                               if epc.metrics_path(m, False) == 'pair'])
def test_maps_points_match_pair_kernel_sums(ctx, monkeypatch, M):
  """K6e's point values (twin network) against ens_pair_kernel's per-field
  sums of the same two points.  The skill takes the same operations on both
  paths: one float32 rounding of the sum apart (the pair kernel may fuse a
  point's scaling into that sum).  The mean and the networks round
  differently on the two paths, so the other statistics agree within both
  paths' bounds."""
  case = _case(M)
  _setenv(monkeypatch, {})
  out = run_metrics(ctx, case, False)
  maps = run_maps(ctx, case, False)
  fin = case.finite().reshape(-1, 2).all(axis=1)
  ref = epc.reference(case, False)
  bp = epc.bounds(case, False, 'pair', ref)
  bt = epc.bounds(case, False, 'twin', ref)
  bad = []
  for i, k in enumerate(STATS):
    m = maps[i].astype(np.float64).reshape(-1, 2)
    if k == 'skill':
      tol = 2 * U * np.abs(m).sum(axis=1)
    else:
      tol = (bp[k] + bt[k]).reshape(-1, 2).sum(axis=1) + 2 * U * np.abs(m).sum(axis=1)
    err = np.abs(out[:, i] - m.sum(axis=1))
    for j in np.flatnonzero(fin & ~(err <= tol)):
      bad.append(f'M={M} field={j} ({case.labels[2 * j]}) {k}: pair {out[j, i]!r} '
                 f'maps {m[j].tolist()} err {err[j]:.3g} tol {tol[j]:.3g}')
  _report(bad)


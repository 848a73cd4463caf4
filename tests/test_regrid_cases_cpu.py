"""The seeded conservative-regridding cases (regrid_cases.py) without a GPU:
every case reaches the kernel instance it claims under a model of the host
dispatch, every instance is reached, the float64 reference agrees with the
oracle, the per-cell bound of DESIGN.md K5 holds for a float32 model of the
kernels' tap order and fails for a model that drops a tap, and the NumPy
stand-in agrees with the reference."""
import numpy as np
import pytest

from oracle import wb2_oracle as orc
import regrid_cases as rc


@pytest.fixture(scope='module')
def cases():
  return rc.all_cases()


def test_every_case_reaches_its_claimed_instance(cases):
  wrong = [(c.name, rc.instance(c.lon, c.lat), c.claim) for c in cases
           if rc.instance(c.lon, c.lat) != c.claim]
  assert not wrong
  for c in cases:  # the forced LDG path and unaligned bases take regrid.cu
    ldg = f'LDG DPT{-(-c.lat.n_src // 256)}'
    assert rc.instance(c.lon, c.lat, force_ldg=True) == ldg
    assert rc.instance(c.lon, c.lat, base_offset=4) == ldg


def test_every_instance_is_reached(cases):
  """All 14 instances (TMA G 2 / 4 x DPT 1-4 generic plus NTAP 7 at DPT 3, and
  LDG DPT 1-4) are reachable; G = 4 at DPT 1 and G = 4 with seven taps only
  through a raw CSR, not through any grid pair of the cases."""
  table = {}
  for c in cases:
    table.setdefault(c.claim, []).append(c.name)
  print('\n'.join(f'{k:20s} {len(table.get(k, []))} cases'
                  for k in rc.INSTANCES))
  assert set(table) == set(rc.INSTANCES)
  for inst in rc.INSTANCES:
    assert any(c.family == 'inf' for c in cases if c.claim == inst), inst
  grid_reached = {c.claim for c in cases if c.family == 'realistic'}
  assert set(rc.INSTANCES) - grid_reached == {'TMA G4 DPT1 NTAP0',
                                              'TMA G4 DPT3 NTAP7'}


def test_unsupported_and_alignment_rules():
  lon, lat = rc.raw_pair('raw-nlat1024')
  lat1025 = rc.raw_csr(1025, [(np.array([0, 1]), np.ones(2))])
  assert rc.instance(lon, lat1025) == 'unsupported'
  assert rc.instance(lon, lat) == 'TMA G2 DPT4 NTAP0'
  # a field stride that is not a multiple of 4 floats takes regrid.cu
  assert rc.instance(lon, lat, src_stride=lon.n_src * 1024 + 2) == 'LDG DPT4'
  for off in (4, 8, 12):
    assert rc.instance(lon, lat, base_offset=off) == 'LDG DPT4'


def test_spikes_sit_where_staging_goes_wrong(cases):
  for c in cases:
    if not c.name.endswith('/spikes'):
      continue
    b, d = np.nonzero(c.x.any(0))
    nlat, nlon = c.lat.n_src, c.lon.n_src
    dpt = -(-nlat // 256)
    assert (b == 0).any() or (b == nlon - 1).any(), c.name  # the seam
    assert (d == 0).any() and (d == nlat - 1).any(), c.name
    assert (d >= 256 * (dpt - 1)).any(), c.name
    # footprints within one field are pairwise disjoint: no target cell taps
    # two spikes
    for f in range(c.nfield):
      seen = np.zeros((c.lon.n_tgt, c.lat.n_tgt), np.int64)
      for bb, dd in zip(*np.nonzero(c.x[f])):
        ia = np.zeros(c.lon.n_tgt, np.int64)
        ic = np.zeros(c.lat.n_tgt, np.int64)
        ia[list(rc._footprint(c.lon, bb))] = 1
        ic[list(rc._footprint(c.lat, dd))] = 1
        seen += np.outer(ia, ic)
      assert seen.max() == 1, c.name


def _oracle_grid(g):
  return orc.Grid(np.asarray(g.longitudes), np.asarray(g.latitudes),
                  periodic=g.periodic, includes_poles=g.includes_poles)


@pytest.mark.parametrize('name', [n for n, *_ in rc._pairs()])
def test_reference_equals_oracle_on_finite_inputs(name):
  """The oracle is the reference's dense float32 contraction: a sum over all
  nlon_s and nlat_s terms, so within (nlon_s + nlat_s + 2) u (A + |T|) / C."""
  c = rc.get_case(name)
  s, t = rc.grid_pair(name)
  x = c.x[:3]
  want = orc.conservative_regrid(x, _oracle_grid(s), _oracle_grid(t))
  ref = rc.reference(c.lon, c.lat, x)
  np.testing.assert_array_equal(np.isnan(want), np.isnan(ref.want))
  fin = np.isfinite(ref.want)
  k = c.lon.n_src + c.lat.n_src + 2
  ref.C[~fin] = 1.0
  tol = rc.U * np.abs(ref.want) + k * rc.U * (ref.A + np.abs(ref.T)) / ref.C
  err = np.abs(want.astype(np.float64) - ref.want)
  assert (err[fin] <= tol[fin]).all()


@pytest.mark.parametrize('name', [n for n, *_ in rc._pairs()])
def test_float32_tap_order_model_passes_the_bound(name):
  c = rc.get_case(name)
  got = rc.model_f32(c.lon, c.lat, c.x)
  assert not rc.violations(got, c.ref)
  fin = np.isfinite(c.ref.want) & (c.ref.bound > 0)  # bound 0: exact zeros
  ratio = np.abs(got - c.ref.want)[fin] / c.ref.bound[fin]
  assert ratio.max() < 0.5  # the bound is not loose by orders of magnitude
  if name != '1440x721-1440x721':  # one tap per cell: exact
    assert ratio.max() > 1e-3


# (grid pair, share of z500 cells the bound flags, share the old check flags)
DROP = [('1440x721-240x121', 0.8, 0.45), ('1440x721-64x32', 0.45, 0.4),
        ('720x361-240x121', 0.95, 0.9), ('360x181-240x121', 0.95, 0.9)]


@pytest.mark.parametrize('name,bound_min,old_max', DROP)
def test_bound_catches_a_dropped_tap_the_old_check_misses(name, bound_min,
                                                          old_max):
  """Drop every longitude target's smallest-weight tap.  On the z500 field
  the per-cell bound flags most cells; the old rtol = 1e-5, atol = 2e-6 check
  lets most of them through (at 0.25 -> 1.5 degrees: 84 % flagged by the
  bound, 41 % by the old check)."""
  c = rc.get_case(name)
  x = c.x[:1]  # z500
  ref = rc.reference(c.lon, c.lat, x)
  got = rc.model_f32(c.lon, c.lat, x, drop_smallest=True)
  fin = np.isfinite(ref.want)
  err = np.abs(got - ref.want)[fin]
  by_bound = (err > ref.bound[fin]).mean()
  by_old = (err > 2e-6 + 1e-5 * np.abs(ref.want[fin])).mean()
  print(f'{name}: bound flags {by_bound:.3f}, old check {by_old:.3f}')
  assert rc.violations(got, ref)
  assert by_bound >= bound_min and by_old <= old_max and by_bound > by_old


def _stand_in(c):
  import fake_ctx
  ctx = fake_ctx.FakeContext()
  x = np.ascontiguousarray(c.x)
  out = np.zeros((c.nfield, c.lon.n_tgt, c.lat.n_tgt), np.float32)
  ns, nt = x[0].size, out[0].size
  ctx.regrid_conservative(x.ctypes.data, out.ctypes.data, c.nfield, ns, nt,
                          c.lon, c.lat)
  return out


def test_stand_in_agrees_with_the_reference(cases):
  for c in cases:
    if c.x.size > 3e7:
      continue
    got = _stand_in(c)
    ref = c.ref
    assert not rc.violations(got, ref, zero_exact=c.zero_exact,
                             value_exact=c.value_exact), c.name
    fin = np.isfinite(ref.want)
    with np.errstate(invalid='ignore', divide='ignore'):
      tol = rc.U * np.abs(ref.want) + 1e-12 * ref.A / ref.C
    assert (np.abs(got[fin] - ref.want[fin]) <= tol[fin]).all(), c.name


def test_bad_csr_pairs_are_malformed_as_claimed():
  for name, lon, lat in rc.bad_csr_pairs():
    bad = False
    for m in (lon, lat):
      for i in range(m.n_tgt):
        cols = rc.taps(m, i)[0]
        bad |= bool((np.diff(cols) <= 0).any())
    assert bad, name

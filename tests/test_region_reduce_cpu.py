"""The cases of region_cases.py reach what they claim, their sums are exact,
and their float64 reference is the stand-in's (fake_ctx.FakeContext), on the
CPU.  test_region_reduce_gpu.py holds the kernels to these references."""
import numpy as np
import pytest

import fake_ctx
import region_cases as rc

EXACT = rc.exact_cases()
MANY = rc.many_field_cases()


def _plans(case):
  return [rc.plan(case, env) for env in case.env]


def test_every_coverage_item_is_reached():
  """Each item of region_cases.COVERAGE is claimed by at least one case, and
  every claim holds under the dispatch model.  The table printed with -s
  lists the cases behind every item."""
  reached = {k: [] for k in rc.COVERAGE}
  for name, case in EXACT.items():
    plans = _plans(case)
    for item in case.covers:
      assert item in rc.COVERAGE, (name, item)
      assert rc.COVERAGE[item](case, plans[0], plans), (
          f'{name} does not reach {item}: {plans[0]}')
      reached[item].append(name)
  missing = [k for k, v in reached.items() if not v]
  assert not missing, missing
  for k, v in reached.items():
    print(f'{k:28s} {", ".join(v)}')


# path, launches, region chunks, bands per chunk, lane rounds per half row
EXPECTED = {
    'k1_tma_r1_c128_plain_sk0': ('tma', 2),
    'k1_tma_r181_c128_clim_sk1': ('tma', 2),
    'k1_tma_stage_fallback': ('ldg', 2),
    'k1_seg_r8_sk0': ('tma_seg', 2, 1, (5,), (1, 1)),
    'k1_seg_r8_sk1': ('tma_seg', 2, 1, (5,), (1, 1)),
    'k1_seg_r9_sk0': ('tma_seg', 2, 1, (5,), (1, 1)),
    'k1_seg_r9_sk1': ('tma_seg', 6, 2, (5, 3), (1, 1)),
    'k1_seg_r16_sk0': ('tma_seg', 2, 1, (5,), (1, 1)),
    'k1_seg_r16_sk1': ('tma_seg', 6, 2, (5, 5), (1, 1)),
    'k1_seg_r17_sk0': ('tma_seg', 6, 2, (5, 3), (1, 1)),
    'k1_seg_r17_sk1': ('tma_seg', 9, 3, (5, 5, 4), (1, 1)),
    'k1_seg_r32_sk0': ('tma_seg', 6, 2, (5, 5), (1, 1)),
    'k1_seg_r32_sk1': ('tma_seg', 12, 4, (5, 5, 5, 5), (1, 1)),
    'k1_seg_128_bands': ('tma_seg', 2, 1, (128,), (1, 1)),
    'k1_seg_129_bands': ('ldg', 2),
    'k1_seg_second_round': ('tma_seg', 6, 2, (6, 4), (2, 1)),
    'k1_seg_too_many_spans': ('ldg', 2),
    'k1_seg_zero_rows': ('tma_seg', 2, 1, (9,), (1, 1)),
    'k1_ldg_odd_offsets': ('ldg', 2),
    'k2_pair_m64': ('pair', 2),
    'k2_odd_offset': ('twin', 2),
    'k2_scalar_m33': ('scalar', 2),
    'k2b_m128': ('big', 2),
    'host_det_tma_groups': ('tma', 16),
    'host_ens_groups': ('twin', 6),
}


@pytest.mark.parametrize('name', list(EXPECTED))
def test_dispatch_model(name):
  """Path, launch count, region chunks (3 launches each, 2 for a single chunk
  that writes the output directly), bands and span rounds of the cases that
  sit at a dispatch limit."""
  p = rc.plan(EXACT[name])
  want = EXPECTED[name]
  assert (p.path, p.launches) == want[:2], p
  if p.path == 'tma_seg':
    assert (p.chunks, p.bands, p.rounds) == want[2:], p


def test_dispatch_model_forced_paths():
  seg = EXACT['k1_seg_r17_sk0']
  assert rc.plan(seg, {'WB2_DET_PATH': 'ldg'}).path == 'ldg'
  pair = EXACT['k2_pair_m16']
  assert rc.plan(pair, {'WB2_ENS_PATH': 'scalar'}).path == 'twin'
  assert rc.plan(pair, {'WB2_ENS_PATH': 'scalar',
                        'WB2_ENS_SORT': 'exact'}).path == 'scalar'
  # the bands / span limits themselves
  # 31 one-column segments + the rest of the half row: 32 spans, one round
  assert rc.seg_spans(128, np.r_[np.arange(0, 32), 128])[0] == 32
  # 33 pieces: no span length fits 32 lanes, the second round takes S = 1
  assert rc.seg_spans(128, np.r_[np.arange(0, 33), 128])[0] == 64
  assert rc.seg_spans(256, np.r_[np.arange(0, 64), 256])[0] == 64
  assert rc.seg_spans(256, np.r_[np.arange(0, 65), 256]) is None


@pytest.mark.parametrize('name', list(EXACT) + list(MANY))
def test_bit_budget(name):
  """Every accumulator of every path the case runs on spans <= 24 bits
  (float32) or <= 53 bits (float64): the kernels' sums are exact, so the GPU
  test may require bit equality."""
  case = EXACT.get(name) or MANY[name]
  for env in case.env:
    b = rc.bit_budget(case, env)
    assert b['f64_region'] <= 53, b
    for k in ('f32_rowseg', 'f32_band'):
      if k in b:
        assert b[k] <= 24, (env, k, b)


def _fake_run(case):
  from weatherbench2_b200 import _lib
  ctx = fake_ctx.FakeContext()
  keep = {k: np.ascontiguousarray(v) for k, v in case.buffers.items()}
  a = {k: v.ctypes.data for k, v in keep.items()}
  cell = None
  if case.cell_w is not None:
    keep['cell'] = np.ascontiguousarray(case.cell_w)
    cell = keep['cell'].ctypes.data
  spec = case.weight_spec(cell)
  o = case.offsets
  dt = _lib.F32 if case.dtype == np.float32 else _lib.F64
  if case.kind == 'energy':
    out = np.zeros((case.nfield, case.nregion, 4, case.nmember))
    ctx.energy_score(a['x'], a['t'], dt, case.nmember, case.member_stride,
                     o['x'], o['t'], spec, out.ctypes.data)
    return out
  out = np.zeros((case.nfield, case.nregion, 10))
  if case.kind == 'det':
    ctx.det_metrics(a['f'], a['t'], a.get('c'), dt, o['f'], o['t'], o.get('c'),
                    spec, case.skipna, out.ctypes.data)
  elif case.kind == 'vector':
    ctx.det_metrics_vector(a['f'], a['fv'], a['t'], a['tv'], dt, o['f'],
                           o['fv'], o['t'], o['tv'], spec, case.skipna,
                           out.ctypes.data)
  else:
    ctx.ens_metrics(a['x'], a['t'], dt, case.nmember, case.member_stride,
                    o['x'], o['t'], spec, case.skipna, out.ctypes.data)
  return out


@pytest.mark.parametrize('name', list(EXACT))
def test_reference_is_the_stand_in(name):
  """The dense reference equals FakeContext bit for bit, NaN placement
  included (the CPU operator suites rely on the stand-in)."""
  case = EXACT[name]
  want, got = rc.reference(case), _fake_run(case)
  mask = rc.exact_slots(case)
  if mask is None:
    np.testing.assert_array_equal(want, got)
  else:  # sums of rounded point values depend on the summation order
    np.testing.assert_array_equal(want[..., mask], got[..., mask])
    np.testing.assert_allclose(want[..., ~mask], got[..., ~mask], rtol=1e-13,
                               atol=1e-13)


@pytest.mark.parametrize('name', list(EXACT) + list(MANY))
def test_sentinels_lie_outside_every_slab(name):
  """Every element no slab reads is NaN, including one before the first and
  one after the last slab; every slab lies inside its buffer."""
  case = EXACT.get(name) or MANY[name]
  for op, buf in case.buffers.items():
    covered = np.zeros(buf.size, bool)
    idx = (np.arange(case.nrow)[:, None] * case.row_stride +
           np.arange(case.ncol)[None, :]).reshape(-1)
    for s in case.slabs[op]:
      assert s >= 1 and s + idx[-1] + 1 < buf.size, (op, s)
      covered[s + idx] = True
    assert np.isnan(buf[~covered]).all(), op
    assert not covered[0] and not covered[-1]
    if case.row_stride > case.ncol:
      assert (~covered).sum() > case.nfield * (case.nrow - 1)
  # the offsets are the slab starts the kernels are given
  for op, off in case.offsets.items():
    assert set(off.tolist()) <= set(case.slabs[op].tolist())


def test_nan_and_dead_cells_on_every_path():
  """Every path runs, without skipna, on a case whose reference is NaN / Inf
  in some regions of a field and finite in others (a kernel that drops NaN,
  or skips a cell by the union of the regions, fails), and, under zero_skip,
  on a case with a row or a whole segment that no region weighs."""
  nan_paths, dead_paths = set(), set()
  for case in list(EXACT.values()) + list(MANY.values()):
    for env in case.env:
      path = rc.plan(case, env).path
      if not case.skipna and rc.nan_per_region(case):
        nan_paths.add(path)
      dead = (case.dense_w() == 0).all(axis=0)
      if case.zero_skip and (dead.all(axis=1).any() or dead.all(axis=0).any()):
        dead_paths.add(path)
  every = {'ldg', 'tma', 'tma_seg', 'pair', 'twin', 'scalar', 'big', 'energy'}
  assert every <= nan_paths, every - nan_paths
  assert every <= dead_paths, every - dead_paths


def test_zero_weight_cells_hold_nan_or_inf():
  """Under zero_skip the cells no region weighs hold NaN / Inf, so a kernel
  that stops skipping them fails."""
  n = 0
  for case in EXACT.values():
    if not case.zero_skip:
      continue
    allzero = (case.dense_w() == 0).all(axis=0)
    if not allzero.any():
      continue
    v = case.fields('x' if 'x' in case.buffers else 'f')
    assert (~np.isfinite(v[..., allzero])).all(), case.name
    n += 1
  assert n >= 10


def test_realistic_family_dispatch():
  """The realistic launches reach TMA-seg (lat_lon, longitude boxes), LDG
  with col_w (lon_lat) and LDG with the fractional land mask."""
  cases = rc.realistic_cases(fake_ctx.FakeContext())
  paths = {c.name: rc.plan(c).path for c in cases}
  assert paths['real_181x360_official_g0'] == 'tma_seg'
  assert paths['real_721x1440_official_g0'] == 'tma_seg'
  assert all(p == 'ldg' for n, p in paths.items() if 'lonlat' in n)
  land = [c for c in cases if c.cell_w is not None and c.kind == 'det']
  assert land and all(paths[c.name] == 'ldg' for c in land)
  assert all(((0 < c.cell_w) & (c.cell_w < 1)).any() for c in land)

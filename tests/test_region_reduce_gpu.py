"""The region-weighted reduction every metric kernel shares
(csrc/region_reduce.cuh) called through `_lib.Context` on the seeded cases of
region_cases.py.

Exact family: inputs and weights on a dyadic grid make every sum exact (the
CPU test proves the bit budget), so every path -- K1 LDG / TMA / TMA-seg, K2
pair / twin / scalar, K2b, K3, the *_host entries -- must equal the float64
reference BIT FOR BIT, NaN pattern included, under every forced path, twice in
a row, in any field order and at any nfield.  A row, segment, region, field or
CTA slot charged to the wrong place fails, however small its weight.

Realistic family: float32 data, cosine latitude weights, the 16 official
regions, a fractional land mask, both layouts, held to
|kernel - ref| <= k u sum |W v| per slot (u = 2^-24) with k derived per path
in `_k_realistic`."""
import numpy as np
import pytest

import region_cases as rc

pytestmark = pytest.mark.gpu

EXACT = rc.exact_cases()
MANY = rc.many_field_cases()
RUNS = [(name, i) for name, c in EXACT.items() for i in range(len(c.env))]


@pytest.fixture(scope='module')
def ctx():
  from weatherbench2_b200 import _lib
  return _lib.default_context(0)


@pytest.fixture(scope='module')
def num_sms():
  import torch
  return torch.cuda.get_device_properties(0).multi_processor_count


def _dev(a):
  import torch
  return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _out_shape(case):
  if case.kind == 'energy':
    return (case.nfield, case.nregion, 4, case.nmember)
  return (case.nfield, case.nregion, 10)


def run(ctx, case, order=None):
  """The raw output of `case` (fields in `order`), and the launches made."""
  import torch
  from weatherbench2_b200 import _lib
  order = np.arange(case.nfield) if order is None else np.asarray(order)
  off = {k: np.ascontiguousarray(v[order]) for k, v in case.offsets.items()}
  dt = _lib.F32 if case.dtype == np.float32 else _lib.F64
  shape = (order.size,) + _out_shape(case)[1:]
  keep = []
  cell = case.cell_w_dev
  if cell is None and case.cell_w is not None:
    keep.append(_dev(case.cell_w))
    cell = keep[-1].data_ptr()
  spec = case.weight_spec(cell)
  before = ctx.launch_count
  if case.host:
    bufs = {k: np.ascontiguousarray(v) for k, v in case.buffers.items()}
    out = np.full(shape, 7.0)
    if case.kind == 'det':
      ctx.det_metrics(bufs['f'].ctypes.data, bufs['t'].ctypes.data,
                      bufs['c'].ctypes.data if case.clim else None, dt,
                      off['f'], off['t'], off.get('c'), spec, case.skipna,
                      out.ctypes.data, host=True)
    else:
      ctx.ens_metrics_host(bufs['x'].ctypes.data, bufs['t'].ctypes.data,
                           case.nmember, case.member_stride, off['x'],
                           off['t'], spec, case.skipna, out.ctypes.data)
    return out, ctx.launch_count - before
  d = {k: _dev(v) for k, v in case.buffers.items()}
  out = torch.full(shape, 7.0, dtype=torch.float64, device='cuda')
  p = {k: v.data_ptr() for k, v in d.items()}
  if case.kind == 'det':
    ctx.det_metrics(p['f'], p['t'], p.get('c'), dt, off['f'], off['t'],
                    off.get('c'), spec, case.skipna, out.data_ptr())
  elif case.kind == 'vector':
    ctx.det_metrics_vector(p['f'], p['fv'], p['t'], p['tv'], dt, off['f'],
                           off['fv'], off['t'], off['tv'], spec, case.skipna,
                           out.data_ptr())
  elif case.kind == 'ens':
    ctx.ens_metrics(p['x'], p['t'], dt, case.nmember, case.member_stride,
                    off['x'], off['t'], spec, case.skipna, out.data_ptr())
  else:
    ctx.energy_score(p['x'], p['t'], dt, case.nmember, case.member_stride,
                     off['x'], off['t'], spec, out.data_ptr())
  ctx.synchronize()
  return out.cpu().numpy(), ctx.launch_count - before


def check_exact(case, got, want, vals=None, what=''):
  mask = rc.exact_slots(case)
  if mask is None:
    np.testing.assert_array_equal(got, want, what)
    return
  np.testing.assert_array_equal(got[..., mask], want[..., mask], what)
  bad = ~mask
  g, w = got[..., bad], want[..., bad]
  np.testing.assert_array_equal(np.isnan(g), np.isnan(w), what + ' NaN')
  bound = rc.ens_bound(case, vals)[..., bad]
  ok = np.isnan(w) | (np.abs(g - w) <= bound)
  assert ok.all(), (f'{what}: {np.argwhere(~ok)[:5]} got {g[~ok][:5]} want '
                    f'{w[~ok][:5]} bound {bound[~ok][:5]}')


@pytest.mark.parametrize('name,variant', RUNS,
                         ids=[f'{n}-{i}' for n, i in RUNS])
def test_exact_family(ctx, num_sms, monkeypatch, name, variant):
  case = EXACT[name]
  env = case.env[variant]
  if num_sms != rc.NUM_SMS and any(c.startswith('tma_') for c in case.covers):
    pytest.skip(f'grid-regime case assumes {rc.NUM_SMS} SMs, device has {num_sms}')
  for k, v in env.items():
    monkeypatch.setenv(k, v)
  plan = rc.plan(case, env)
  vals = rc.point_values(case)
  want = rc.reference(case, vals)
  if case.stage_mb:
    from weatherbench2_b200 import _lib
    monkeypatch.setenv('WB2_STAGE_MB', str(case.stage_mb))
    own = _lib.Context(0)  # the staging buffer only grows: start from none
    try:
      got, n = run(own, case)
      again, _ = run(own, case)
    finally:
      own.close()
  else:
    got, n = run(ctx, case)
    again, _ = run(ctx, case)
  check_exact(case, got, want, vals, f'{name} {env}')
  assert n == plan.launches, (n, plan)
  np.testing.assert_array_equal(again, got)


@pytest.mark.parametrize('name', list(MANY))
def test_field_order_and_nfield(ctx, name):
  """Per-field results do not depend on which other fields share the launch:
  prefixes of 1, 131, 132, 133 and all fields and a permutation give the
  reference's rows bit for bit in every exact slot (the rows per CTA, and so
  the float64 order of the rounded K2 slots, follow nfield).  k1_tma_scratch
  is nrow = 1 with 20 000 fields and 32 regions: the TMA partials are ~413 MB
  there."""
  case = MANY[name]
  vals = rc.point_values(case)
  want = rc.reference(case, vals)
  perm = np.random.RandomState(1).permutation(case.nfield)
  for order in ([0], np.arange(131), np.arange(132), np.arange(133), perm,
                np.arange(case.nfield)):
    order = np.asarray(order)
    got, _ = run(ctx, case, order)
    sub = rc.select_fields(case, order)
    check_exact(sub, got, want[order], rc.point_values(sub),
                f'{name} n={order.size}')


# ---- realistic family ------------------------------------------------------------
def _k_realistic(case, plan):
  """Multiple of u * sum |W v| that bounds |kernel - ref| per slot.

  A point value v is formed in float32 from float32 inputs: d = f - t, fa, ta
  carry one rounding, d^2 and fa * ta three, so |v32 - v| <= 3 u |v|.  The
  non-separable weight col_w * cell_w is one float32 product (u) and wc * v
  another (u).  LDG / TMA / K2 sum the n cells of one (row, segment) -- for
  TMA half a row, n <= ncol -- in float32: (n - 1) u sum |wc v|; the float64
  weight and region sums add ~1e-16 relative.  So k = n + 5.
  TMA-seg instead sums a lane's span of S <= n cells (S u), scales it by the
  float32 row factor and accumulates up to 16 rows (u + 16 u), multiplies by
  the float32 pattern * segment weight (row_c, pattern and seg_w rounded to
  float32, their product and the scaling: 5 u) and adds 32 lanes x 2 spans in
  a float32 butterfly (64 u): k = 3 + S + 17 + 5 + 64 <= n + 89.
  K2 point values (10 members): mean, 1/M, 1/(M-1) and the member sums,
  bounded by (2 M + 8) u A^p as in region_cases.ens_bound."""
  n = int(np.diff(case.seg_start).max())
  if plan.path == 'tma_seg':
    return n + 89
  return n + 5


@pytest.fixture(scope='module')
def realistic(ctx):
  return rc.realistic_cases(ctx)


def test_realistic_family(ctx, realistic):
  for case in realistic:
    plan = rc.plan(case)
    vals = rc.point_values(case)
    want = rc.reference(case, vals)
    got, n = run(ctx, case)
    assert n == plan.launches, (case.name, n, plan)
    W = np.abs(case.dense_w())
    tot = W.reshape(case.nregion, -1).sum(axis=1)[None]
    exact_counts = (case.col_w is None and case.cell_w is None and
                    plan.path != 'tma_seg')
    if case.kind == 'ens':
      bound = rc.ens_bound(case, vals)
      bound[..., 5:] = ((1e-13 if exact_counts else _k_realistic(case, plan) * rc.U) *
                        tot[..., None])
    else:
      k = _k_realistic(case, plan) * rc.U
      bound = np.zeros_like(want)
      names = ['d2', 'ad', 'd'] + (['fata', 'fa2', 'ta2'] if case.clim else [])
      cnt = {'d2': 6, 'fata': 7, 'fa2': 8, 'ta2': 9}
      for j, nm in enumerate(names):
        a = np.abs(vals[nm]).reshape(case.nfield, -1)
        bound[..., j] = k * (a @ W.reshape(case.nregion, -1).T)
        # weight sums: exact float32 cell counts, one float64 weight product
        # per (row, segment), unless col_w / cell_w or TMA-seg's float32
        # weights enter
        if nm in cnt:
          bound[..., cnt[nm]] = (1e-13 if exact_counts else k) * tot
    err = np.abs(got - want)
    ok = err <= bound + 1e-300
    assert ok.all(), (case.name, plan.path, np.argwhere(~ok)[:5],
                      got[~ok][:5], want[~ok][:5], bound[~ok][:5])


# ---- the zero_skip sign contract ---------------------------------------------------
def test_zero_skip_rejects_negative_weights(ctx):
  from weatherbench2_b200 import _lib
  case = EXACT['k1_negative_weights']
  spec = case.weight_spec()
  spec.zero_skip = True
  buf = ctx.malloc(1 << 16)
  off = np.zeros(1, np.int64)
  try:
    before = ctx.launch_count
    with pytest.raises(_lib.Wb2Error, match='non-negative'):
      ctx.det_metrics(buf, buf, None, _lib.F32, off, off, None, spec, False,
                      buf)
    with pytest.raises(_lib.Wb2Error, match='non-negative'):
      ctx.ens_metrics(buf, buf, _lib.F32, 4, 8, off, off, spec, False, buf)
    assert ctx.launch_count == before
    spec.zero_skip = False  # the same weights are accepted without zero_skip
    ctx.det_metrics(buf, buf, None, _lib.F32, off, off, None, spec, False,
                    buf + (1 << 15))
  finally:
    ctx.synchronize()
    ctx.free(buf)

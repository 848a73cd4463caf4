"""The climatology kernels (csrc/climatology.cu, csrc/climatology_quantile.cu)
called through `_lib.Context` directly, on generated index tables
(climatology_tables.py) at the shapes and holes the operators never produce,
against the float64 NumPy interpretations of the same entries
(test_climatology_abi_cpu.py pins those to the oracles).

Reached here and nowhere else: the quantile kernel's fallback to 4, 2 and 1
cells per CTA near 8192 samples per window, 16 quantiles, window 3, 512
stacked years, day axes shorter than the window, uneven hours, partial CTAs,
SEEPS samples exactly at the threshold and absent stacked years; the mean /
std kernel at 1400 days, with idle day lanes, with empty slots, and with a
large-mean field whose first table entries are missing; both host entries
with one cell per band, a band count that does not divide the cells, and no
step at all; and every argument error of both entries."""
import numpy as np
import pytest

from climatology_tables import make_tables
from test_climatology_abi_cpu import fake_moments, fake_quantile

pytestmark = pytest.mark.gpu

RTOL = 2e-6
SPREAD_ATOL = 1e-6  # times the max - min of the cell's series
F32, F64 = np.float32, np.float64


@pytest.fixture(scope='module')
def ctx():
  from weatherbench2_b200 import _lib
  return _lib.default_context(0)


def _code(x):
  from weatherbench2_b200 import _lib
  return _lib.F32 if x.dtype == np.float32 else _lib.F64


def _cell_budget(plan, x, out_rows):
  """Device bytes the host entries stage per cell (clim_stream_host): the
  span of referenced time rows, the resampled days and the outputs."""
  if plan.nres:
    live = plan.res_count > 0
    lo = plan.res_start[live]
    hi = plan.res_start[live] + plan.res_count[live] - 1
  else:
    idx = np.concatenate([plan.items.ravel(), plan.fill.ravel()])
    lo = hi = idx[idx >= 0]
  rows = int(hi.max() - lo.min() + 1) if lo.size else 0
  return rows * x.itemsize + plan.nres * 4 + out_rows * 4


def _bands(plan, x, out_rows, cells_per_band):
  """(budget, number of bands) for `cells_per_band` cells per band."""
  budget = 2 * _cell_budget(plan, x, out_rows) * cells_per_band
  return budget, -(-x.shape[1] // cells_per_band)


def gpu_quantile(ctx, plan, x, qs, thr=None, cells_per_band=None):
  """The kernel's (out, dry fraction): device tensors, or the host entry with
  `cells_per_band` cells per band."""
  import torch
  ntime, ncell = x.shape
  oshape = (plan.nhour, len(qs), plan.nday_out, ncell)
  dshape = (plan.nhour, plan.nday_out, ncell)
  before = ctx.launch_count
  if cells_per_band is None:
    xd = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    out = torch.full(oshape, 7.0, device='cuda')  # every value is written
    dry = torch.full(dshape, 7.0, device='cuda') if thr is not None else None
    ctx.climatology_quantile(xd.data_ptr(), _code(x), ntime, ncell, plan, qs,
                             thr, out.data_ptr(),
                             dry.data_ptr() if dry is not None else None)
    bands = 1
    out, dry = out.cpu().numpy(), dry.cpu().numpy() if dry is not None else None
  else:
    out = np.full(oshape, 7.0, np.float32)
    dry = np.full(dshape, 7.0, np.float32) if thr is not None else None
    budget, bands = _bands(plan, x, out.size // max(ncell, 1) +
                           (dry.size // max(ncell, 1) if dry is not None
                            else 0),
                           cells_per_band)
    ctx.climatology_quantile_host(x.ctypes.data, _code(x), ntime, ncell, plan,
                                  qs, thr, budget, out.ctypes.data,
                                  dry.ctypes.data if dry is not None else None)
  if ncell and not plan.nres:  # one launch per band (the resample adds some)
    assert ctx.launch_count - before == bands
  return out, dry


def gpu_moments(ctx, plan, x, stats=('mean', 'std'), cells_per_band=None):
  """{stat: [nhour][nday_out][ncell]} of the mean / std kernel."""
  import torch
  ntime, ncell = x.shape
  shape = (plan.nhour, plan.nday_out, ncell)
  before = ctx.launch_count
  if cells_per_band is None:
    xd = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    out = {s: torch.full(shape, 7.0, device='cuda') for s in stats}
    ptr = {s: out[s].data_ptr() if s in out else None for s in ('mean', 'std')}
    ctx.climatology(xd.data_ptr(), _code(x), ntime, ncell, plan, ptr['mean'],
                    ptr['std'])
    bands = 1
    out = {s: v.cpu().numpy() for s, v in out.items()}
  else:
    out = {s: np.full(shape, 7.0, np.float32) for s in stats}
    ptr = {s: out[s].ctypes.data if s in out else None
           for s in ('mean', 'std')}
    budget, bands = _bands(plan, x, len(stats) * plan.nhour * plan.nday_out,
                           cells_per_band)
    ctx.climatology_host(x.ctypes.data, _code(x), ntime, ncell, plan, budget,
                         ptr['mean'], ptr['std'])
  if not plan.nres:
    assert ctx.launch_count - before == bands
  return out


def assert_matches(got, want, x, err_msg=''):
  """float32 kernel output against the float64 reference: identical NaN
  masks, rtol 2e-6, atol 1e-6 x the spread of the cell's series."""
  np.testing.assert_array_equal(np.isnan(got), np.isnan(want),
                                err_msg=f'NaN mask {err_msg}')
  finite = np.isfinite(x)
  with np.errstate(invalid='ignore'):
    spread = (np.where(finite, x, -np.inf).max(0) -
              np.where(finite, x, np.inf).min(0)).astype(np.float64)
  spread = np.where(finite.any(0), spread, 0.0)
  ok = np.isnan(want) | (np.abs(got - want) <=
                         RTOL * np.abs(want) + SPREAD_ATOL * spread)
  if not ok.all():
    i = np.unravel_index(np.argmin(ok), ok.shape)
    raise AssertionError(f'{err_msg}: {(~ok).sum()} of {ok.size} values off, '
                         f'first at {i}: got {got[i]!r}, want {want[i]!r}')


# -- quantile / SEEPS kernel ----------------------------------------------------
Q5 = [0.1, 0.25, 0.5, 0.75, 0.9]
# 16: both ends of [0, 1], duplicates, unsorted
Q16 = [1.0, 0.0, 0.5, 0.5, 0.9, 0.1, 2 / 3, 0.25, 0.75, 0.0, 1.0, 0.33, 0.05,
       0.95, 0.999, 0.001]
SEEPS_THR = 0.25e-3  # metres; not representable in float32
BOTH = (F32, F64)

# (id, make_tables kwargs, quantiles, SEEPS threshold or None, dtypes)
QUANTILE_CASES = [
    # nitem x window near 8192: 2 cells per CTA (float32 and float64)
    ('cap_134x61', dict(nitem=134, window_size=61, nday=5, ncell=3,
                        missing=0.05), Q5, None, BOTH),
    # 4 cells per CTA in float32
    ('cap_64x61', dict(nitem=64, window_size=61, nday=5, ncell=5), Q5, None,
     (F32,)),
    # 1 cell per CTA; the count rings at W = 4095 / 8191; the window at cap
    ('cap_2x4095', dict(nitem=2, window_size=4095, nday=4, ncell=2,
                        missing=0.1), Q5, None, (F64,)),
    ('cap_1x8191', dict(nitem=1, window_size=8191, nday=3, ncell=2, nan=0.1),
     Q5, None, BOTH),
    # the rank sort of `load` over 16 chunks, merges of large batches
    ('nitem512_window15', dict(nitem=512, window_size=15, nday=4, ncell=2,
                               kind='ties', nan=0.1), Q5, None, BOTH),
    ('q16_window31', dict(nitem=5, window_size=31, nday=40, ncell=9,
                          missing=0.1), Q16, None, BOTH),
    ('window3', dict(nitem=4, window_size=3, nday=30, ncell=9, missing=0.2),
     Q16, None, BOTH),
    # n = 1, 2, 10 with window 61 in one call; rows some hour lacks
    ('short_uneven_hours', dict(nhour=3, nday=10, hour_nday=[1, 2, 10],
                                nday_out=16, nitem=3, window_size=61, ncell=9),
     Q5, None, BOTH),
    ('n366_window61', dict(nhour=2, nday=366, hour_nday=[366, 365], nitem=3,
                           window_size=61, ncell=7, missing=0.05), Q5, None,
     BOTH),
    ('n1400_window31', dict(nday=1400, nitem=2, window_size=31, ncell=3), Q5,
     None, (F32,)),
    ('ties_signed_zero', dict(nitem=6, nday=20, window_size=15, ncell=9,
                              kind='ties'), Q16, None, BOTH),
    ('offset_nan_fill', dict(nitem=4, nday=25, window_size=31, ncell=9,
                             kind='offset', nan=0.3, nan_cells=(2, 7),
                             fill_missing=0.3), Q5, None, BOTH),
    ('seeps', dict(nhour=2, nitem=4, nday=30, window_size=31, ncell=9,
                   kind='precip', nan=0.1, nan_cells=(3,),
                   absent_years={1: [1]}), [2 / 3], SEEPS_THR, BOTH),
    ('seeps_short_uneven', dict(nhour=2, nitem=3, nday=7, hour_nday=[7, 2],
                                nday_out=9, window_size=61, ncell=9,
                                kind='precip', absent_years={0: [2]}),
     [2 / 3], SEEPS_THR, BOTH),
    ('seeps_resample', dict(nitem=3, nday=20, window_size=15, ncell=7,
                            kind='precip', steps_per_day=4, empty_days=0.2),
     [2 / 3], SEEPS_THR, (F32,)),
    ('quantile_resample', dict(nhour=2, nitem=3, nday=12, hour_nday=[12, 5],
                               window_size=15, ncell=7, steps_per_day=2,
                               empty_days=0.3, nan=0.2), Q5, None, (F32,)),
]


def _case_data(kw, dtype, thr, seed):
  plan, x = make_tables(seed, dtype=dtype, **kw)
  if thr is not None and x.shape[1] >= 3:
    x[::5] = x.dtype.type(thr)  # exactly at the threshold: not dry
    x[:, 0] = 0.0  # a dry cell: dry fraction 1, threshold NaN
    x[:, 1] = 1.0  # a wet cell: dry fraction 0
    x[:, list(kw.get('nan_cells', ()))] = np.nan
  return plan, x


@pytest.mark.parametrize('dtype', BOTH, ids=['f32', 'f64'])
@pytest.mark.parametrize('case', QUANTILE_CASES,
                         ids=[c[0] for c in QUANTILE_CASES])
def test_quantile_kernel_matches_the_reference(ctx, case, dtype):
  _, kw, qs, thr, dtypes = case
  if dtype not in dtypes:
    pytest.skip('not a case of this dtype')
  plan, x = _case_data(kw, dtype, thr, 21)
  want = fake_quantile(plan, x, qs, thr)
  ncell = x.shape[1]
  for cpb in (None, 1 if ncell <= 3 else 2):  # device; host in bands
    got = gpu_quantile(ctx, plan, x, qs, thr, cpb)
    assert_matches(got[0], want[0], x, f'quantiles, bands of {cpb}')
    if thr is not None:
      assert_matches(got[1], want[1], x, f'dry fraction, bands of {cpb}')


@pytest.mark.parametrize('dtype', BOTH, ids=['f32', 'f64'])
@pytest.mark.parametrize('ncell', [0, 1, 7, 9, 19])
def test_quantile_kernel_partial_ctas(ctx, ncell, dtype):
  plan, x = make_tables(22, nhour=2, nday=12, nitem=5, window_size=9,
                        ncell=ncell, missing=0.1, dtype=dtype)
  want = fake_quantile(plan, x, Q5, None) if ncell else None
  for cpb in (None, 2):
    before = ctx.launch_count
    got = gpu_quantile(ctx, plan, x, Q5, None, cpb)
    if ncell == 0:  # nothing to compute, nothing launched
      assert ctx.launch_count == before and got[0].size == 0
    else:
      assert_matches(got[0], want[0], x, f'bands of {cpb}')


@pytest.mark.parametrize('dtype', BOTH, ids=['f32', 'f64'])
def test_quantile_kernel_returns_a_constant_exactly(ctx, dtype):
  plan, x = make_tables(23, nhour=2, nday=20, hour_nday=[20, 9], nitem=4,
                        window_size=31, ncell=9, kind='constant', missing=0.3,
                        dtype=dtype)
  want, _ = fake_quantile(plan, x, Q16)
  for cpb in (None, 3):
    got, _ = gpu_quantile(ctx, plan, x, Q16, None, cpb)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
    assert np.isfinite(got).any()
    np.testing.assert_array_equal(got[np.isfinite(got)], np.float32(3.7))


def test_host_entries_without_any_step(ctx):
  """Every item and fill entry -1: the host entries copy no row at all
  (rows == 0 in clim_stream_host) and return NaN everywhere."""
  plan, x = make_tables(24, nhour=2, nday=6, nitem=3, window_size=5, ncell=5,
                        kind='precip')
  plan.items[:] = -1
  plan.fill[:] = -1
  for cpb in (None, 1):
    out, dry = gpu_quantile(ctx, plan, x, Q5, None, cpb)
    assert np.isnan(out).all()
    out, dry = gpu_quantile(ctx, plan, x, [2 / 3], SEEPS_THR, cpb)
    assert np.isnan(out).all() and np.isnan(dry).all()
    got = gpu_moments(ctx, plan, x, cells_per_band=cpb)
    assert np.isnan(got['mean']).all() and np.isnan(got['std']).all()


# -- mean / std kernel ----------------------------------------------------------
# (id, make_tables kwargs, methods, dtypes)
MOMENT_CASES = [
    # 224 KB of shared memory; an hour of 700 days in the same call
    ('n1400_uneven', dict(nhour=2, nday=1400, hour_nday=[1400, 700], nitem=2,
                          window_size=61, ncell=9, missing=0.1), (0, 1), BOTH),
    # idle day lanes, uneven chunks, heavy wrap; rows the hours lack
    ('short_n_window61', dict(nhour=5, nday=65, hour_nday=[1, 2, 31, 33, 65],
                              nday_out=70, nitem=3, window_size=61, ncell=9,
                              missing=0.1), (0, 1), BOTH),
    # slots without a valid item; ~960 items per slot
    ('empty_slots_960', dict(nitem=960, nday=12, window_size=5, ncell=9,
                             empty_slots=0.3, missing=0.5, nan=0.2), (0, 1),
     (F32,)),
    ('offset_nan_fill', dict(nitem=4, nday=40, window_size=31, ncell=9,
                             kind='offset', nan=0.3, nan_cells=(4,),
                             fill_missing=0.3), (0, 1), BOTH),
    ('ties', dict(nitem=5, nday=33, window_size=15, ncell=9, kind='ties'),
     (0, 1), (F64,)),
    ('resample', dict(nhour=1, nitem=3, nday=20, window_size=15, ncell=7,
                      steps_per_day=4, empty_days=0.2, nan=0.1), (0, 1),
     (F32,)),
]


@pytest.mark.parametrize('dtype', BOTH, ids=['f32', 'f64'])
@pytest.mark.parametrize('method', [0, 1], ids=['explicit', 'fast'])
@pytest.mark.parametrize('case', MOMENT_CASES, ids=[c[0] for c in
                                                    MOMENT_CASES])
def test_moment_kernel_matches_the_reference(ctx, case, method, dtype):
  _, kw, methods, dtypes = case
  if dtype not in dtypes or method not in methods:
    pytest.skip('not a case of this dtype / method')
  plan, x = make_tables(31, method=method, dtype=dtype, **kw)
  want = fake_moments(plan, x)
  for cpb in (None, 2):
    got = gpu_moments(ctx, plan, x, cells_per_band=cpb)
    for i, s in enumerate(('mean', 'std')):
      assert_matches(got[s], want[i], x, f'{s}, bands of {cpb}')


def _leading_gaps(method, dtype, value=None, seed=32):
  """1e5 + 0.5 N over 10 stacked years, window 61, where the first 300
  entries of each hour's table (day-major) are -1 or NaN in cells 0-3, and
  the only finite values of cell 5 come from the fill."""
  plan, x = make_tables(seed, nhour=2, nday=366, hour_nday=[366, 300],
                        nitem=10, window_size=61, ncell=9, kind='offset',
                        method=method, dtype=dtype)
  if value is not None:
    x[:] = value
  for h in range(plan.nhour):
    head = plan.items[h].reshape(-1)[:300]  # a view: -1 in 100, NaN in 200
    head[:100] = -1
    x[head[100:][head[100:] >= 0], :4] = np.nan
  if method == 0:
    filled = np.zeros(x.shape[0], bool)
    filled[plan.fill[plan.fill >= 0]] = True
    x[~filled, 5] = np.nan
  return plan, x


@pytest.mark.parametrize('dtype', BOTH, ids=['f32', 'f64'])
@pytest.mark.parametrize('method', [0, 1], ids=['explicit', 'fast'])
def test_shift_survives_missing_leading_entries(ctx, method, dtype):
  plan, x = _leading_gaps(method, dtype)
  want = fake_moments(plan, x)
  for cpb in (None, 4):
    got = gpu_moments(ctx, plan, x, cells_per_band=cpb)
    for i, s in enumerate(('mean', 'std')):
      assert_matches(got[s], want[i], x, f'{s}, bands of {cpb}')


def test_shift_keeps_a_constant_exact_behind_missing_entries(ctx):
  """Moments around a shift equal to the constant are exactly 0."""
  c = np.float32(1e5 + 0.25)
  plan, x = _leading_gaps(0, F32, value=c)
  for cpb in (None, 4):
    got = gpu_moments(ctx, plan, x, cells_per_band=cpb)
    fin = np.isfinite(got['mean'])
    assert (fin.sum(axis=1) == plan.hour_nday[:, None]).all()
    np.testing.assert_array_equal(got['mean'][fin], c)
    np.testing.assert_array_equal(got['std'][fin], 0.0)


@pytest.mark.parametrize('stats', [('mean',), ('std',), ('mean', 'std')])
def test_moment_kernel_writes_the_requested_statistics(ctx, stats):
  plan, x = make_tables(33, nhour=2, nday=30, hour_nday=[30, 12], nday_out=31,
                        nitem=3, window_size=15, ncell=11, missing=0.1)
  want = dict(zip(('mean', 'std'), fake_moments(plan, x)))
  for cpb in (None, 3):
    got = gpu_moments(ctx, plan, x, stats, cells_per_band=cpb)
    assert set(got) == set(stats)
    for s in stats:
      assert_matches(got[s], want[s], x, f'{s}, bands of {cpb}')


# -- argument errors --------------------------------------------------------------
def _error_calls(ctx, host):
  """Yields (expected message, call) for every bad argument of both entries
  on a small valid table."""
  import torch
  from weatherbench2_b200 import _lib
  plan0, x = make_tables(40, nhour=2, nday=6, nitem=3, window_size=5, ncell=4)
  ntime, ncell = x.shape
  x64 = x.astype(np.float64)
  dev = {} if host else {'x': torch.from_numpy(x).cuda(),
                         'x64': torch.from_numpy(x64).cuda()}
  bufs = [np.zeros((2, 17, 6, ncell), np.float32) for _ in range(3)]
  if not host:
    bufs = [torch.from_numpy(b).cuda() for b in bufs]
  addr = [b.ctypes.data if host else b.data_ptr() for b in bufs]
  xa = x.ctypes.data if host else dev['x'].data_ptr()
  x64a = x64.ctypes.data if host else dev['x64'].data_ptr()

  def plan(**changes):
    p = _lib.ClimatologyPlan(plan0.items.copy(), plan0.fill.copy(),
                             plan0.hour_nday, plan0.out_row.copy(),
                             plan0.nday_out, plan0.window_size, 0)
    for k, v in changes.items():
      setattr(p, k, v)
    return p

  def quant(p, qs=(0.5,), thr=None, dry=False, xp=xa, code=_lib.F32):
    d = addr[1] if dry else None
    if host:
      return lambda: ctx.climatology_quantile_host(
          xp, code, ntime, ncell, p, qs, thr, 1 << 20, addr[0], d)
    return lambda: ctx.climatology_quantile(xp, code, ntime, ncell, p, qs, thr,
                                            addr[0], d)

  def moments(p, xp=xa, code=_lib.F32):
    if host:
      return lambda: ctx.climatology_host(xp, code, ntime, ncell, p, 1 << 20,
                                          addr[0], addr[2])
    return lambda: ctx.climatology(xp, code, ntime, ncell, p, addr[0], addr[2])

  bad_items = plan0.items.copy()
  bad_items[1, 2, 0] = ntime
  low_items = plan0.items.copy()
  low_items[0, 0, 1] = -2
  bad_fill = plan0.fill.copy()
  bad_fill[1, 1] = ntime
  bad_row = plan0.out_row.copy()
  bad_row[0, 3] = plan0.nday_out
  dup_row = plan0.out_row.copy()
  dup_row[1, 4] = dup_row[1, 3]
  resampled = dict(nres=ntime, res_start=np.arange(ntime, dtype=np.int64),
                   res_count=np.ones(ntime, np.int32))
  for entry in (quant, moments):
    yield 'window_size', entry(plan(window_size=4))
    yield 'window_size', entry(plan(window_size=1))
    yield 'items', entry(plan(items=bad_items))
    yield 'items', entry(plan(items=low_items))
    yield 'fill', entry(plan(fill=bad_fill))
    yield 'out_row', entry(plan(out_row=bad_row))
    yield 'out_row', entry(plan(out_row=dup_row))
    yield 'nres', entry(plan(**resampled), xp=x64a, code=_lib.F64)
  yield 'nquantile', quant(plan(), qs=())
  yield 'nquantile', quant(plan(), qs=np.full(17, 0.5))
  yield r'quantiles\[1\]', quant(plan(), qs=(0.5, np.nan))
  yield r'quantiles\[0\]', quant(plan(), qs=(1.5,))
  yield r'nitem \* window_size', quant(plan(window_size=2731))
  yield 'dry_fraction', quant(plan(), thr=SEEPS_THR, dry=False)
  yield 'dry_fraction', quant(plan(), thr=None, dry=True)


@pytest.mark.parametrize('host', [False, True], ids=['device', 'host'])
def test_argument_errors_name_the_argument_and_launch_nothing(ctx, host):
  from weatherbench2_b200 import _lib
  n = 0
  for msg, call in _error_calls(ctx, host):
    before = ctx.launch_count
    with pytest.raises(_lib.Wb2Error, match=msg):
      call()
    assert ctx.launch_count == before, msg
    n += 1
  assert n == 23

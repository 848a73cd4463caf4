"""The NumPy interpretations of the climatology entries
(fake_ctx_climatology.py, fake_ctx_climatology_quantile.py) against the
hand-pinned float64 oracles, window by window, on generated index tables
(climatology_tables.py) that `utils._plan` never produces: day axes shorter
than the window (slots repeat), uneven hours, absent stacked years, an hour
without any item, NaN items rescued by the fill, resampled days without data.
The GPU tests (test_climatology_abi_gpu.py) hold the kernels to these fakes,
so this file is what makes them a trustworthy reference there."""
import numpy as np
import pytest

import climatology_oracle as co
import climatology_quantile_oracle as cq
from climatology_tables import make_tables
from fake_ctx_climatology import ClimatologyFakeContext
from fake_ctx_climatology_quantile import QuantileFakeContext
from weatherbench2_b200 import _lib


def _dtype_code(x):
  return _lib.F32 if x.dtype == np.float32 else _lib.F64


def fake_moments(plan, x):
  """(mean, std) [nhour][nday_out][ncell] float32 of the fake."""
  ntime, ncell = x.shape
  shape = (plan.nhour, plan.nday_out, ncell)
  mean, std = np.empty(shape, np.float32), np.empty(shape, np.float32)
  x = np.ascontiguousarray(x)
  ClimatologyFakeContext._climatology(  # pylint: disable=protected-access
      x.ctypes.data, _dtype_code(x), ntime, ncell, plan, mean.ctypes.data,
      std.ctypes.data)
  return mean, std


def fake_quantile(plan, x, qs, seeps_threshold=None):
  """(out [nhour][nq][nday_out][ncell], dry fraction [nhour][nday_out][ncell]
  or None) float32 of the fake."""
  ntime, ncell = x.shape
  out = np.empty((plan.nhour, len(qs), plan.nday_out, ncell), np.float32)
  dry = (np.empty((plan.nhour, plan.nday_out, ncell), np.float32)
         if seeps_threshold is not None else None)
  x = np.ascontiguousarray(x)
  QuantileFakeContext._quantile(  # pylint: disable=protected-access
      x.ctypes.data, _dtype_code(x), ntime, ncell, plan, qs, seeps_threshold,
      out.ctypes.data, dry.ctypes.data if dry is not None else 0)
  return out, dry


def _source(plan, x, precision):
  """The series the tables index: x, or its daily resample in `precision`."""
  if not plan.nres:
    return x
  src = np.full((plan.nres, x.shape[1]), np.nan)
  for i in range(plan.nres):
    c, s = int(plan.res_count[i]), int(plan.res_start[i])
    if c:
      with co._quiet():  # pylint: disable=protected-access
        src[i] = np.nanmean(x[s:s + c].astype(np.float64), axis=0)
  return src.astype(precision)


def _window(plan, src, h, d):
  """(tap, stacked year, cell) samples of day slot d of hour h, the day-365
  fill applied, only the hour's stacked years (columns with some step)."""
  n = int(plan.hour_nday[h])
  half = plan.window_size // 2
  it = plan.items[h, (d + np.arange(-half, half + 1)) % n]
  vals = np.where((it >= 0)[..., None], src[np.maximum(it, 0)], np.nan)
  f = plan.fill[h]
  fv = np.where((f >= 0)[:, None], src[np.maximum(f, 0)], np.nan)
  vals = np.where(np.isnan(vals), fv[None], vals)
  return vals[:, (plan.items[h, :n] >= 0).any(axis=0)]


def _assert_float32_of(got, want, err_msg=''):
  np.testing.assert_array_equal(np.isnan(got), np.isnan(want), err_msg=err_msg)
  np.testing.assert_allclose(got, want, rtol=1e-6, atol=1e-12,
                             err_msg=err_msg)


# (id, make_tables kwargs): small tables at the shapes the operators never make
TABLES = [
    ('n1_n2_n10_window31', dict(nhour=3, nday=10, hour_nday=[1, 2, 10],
                                nday_out=12, window_size=31, nitem=3)),
    ('n1_n2_n10_window61', dict(nhour=3, nday=10, hour_nday=[10, 1, 2],
                                nday_out=14, window_size=61, nitem=2,
                                missing=0.2)),
    ('absent_year_columns', dict(nhour=2, nday=12, nitem=4, window_size=7,
                                 absent_years={1: [0, 2]}, missing=0.1)),
    ('hour_without_items', dict(nhour=2, nday=9, nitem=3, window_size=5,
                                absent_years={0: [0, 1, 2]})),
    ('fill_rescues_nan', dict(nday=15, nitem=3, window_size=9, nan=0.35,
                              missing=0.2, fill_missing=0.3)),
    ('resample_with_empty_days', dict(nhour=1, nday=11, nitem=2, window_size=5,
                                      steps_per_day=3, empty_days=0.2,
                                      nan=0.2)),
    ('float64_ties', dict(nday=8, nitem=3, window_size=5, kind='ties',
                          dtype=np.float64, nan_cells=(1,))),
]


@pytest.mark.parametrize('kw', [t[1] for t in TABLES], ids=[t[0] for t in
                                                             TABLES])
def test_fake_moments_match_the_oracle_window_by_window(kw):
  plan, x = make_tables(3, **kw)
  mean, std = fake_moments(plan, x)
  src = _source(plan, x, np.float64).astype(np.float64)
  w = co.window_weights(plan.window_size)
  produced = np.zeros(mean.shape, bool)
  for h in range(plan.nhour):
    for d in range(int(plan.hour_nday[h])):
      win = _window(plan, src, h, d).astype(np.float64).swapaxes(0, 1)
      r = plan.out_row[h, d]
      produced[h, r] = True
      for stat, got in (('mean', mean), ('std', std)):
        _assert_float32_of(got[h, r], co.weighted_stat(win, w, stat),
                           (stat, h, d))
  assert np.isnan(mean[~produced]).all() and np.isnan(std[~produced]).all()


@pytest.mark.parametrize('kw', [t[1] for t in TABLES], ids=[t[0] for t in
                                                             TABLES])
def test_fast_fake_matches_the_smoothed_groupby_oracle(kw):
  kw = dict(kw, method=1)
  plan, x = make_tables(4, **kw)
  mean, std = fake_moments(plan, x)
  src = _source(plan, x, np.float64).astype(np.float64)
  for h in range(plan.nhour):
    n = int(plan.hour_nday[h])
    it = plan.items[h, :n]
    vals = np.where((it >= 0)[..., None], src[np.maximum(it, 0)], np.nan)
    with co._quiet():  # pylint: disable=protected-access
      per_slot = {'mean': np.nanmean(vals, axis=1),
                  'std': np.nanstd(vals, axis=1)}
    for stat, got in (('mean', mean), ('std', std)):
      want = co.smooth_dayofyear(per_slot[stat], plan.window_size)
      _assert_float32_of(got[h, plan.out_row[h, :n]], want, (stat, h))


QS = [0.0, 0.1, 0.5, 2 / 3, 0.9, 1.0]


@pytest.mark.parametrize('kw', [t[1] for t in TABLES], ids=[t[0] for t in
                                                             TABLES])
def test_fake_quantiles_match_the_oracle_window_by_window(kw):
  plan, x = make_tables(5, **kw)
  out, _ = fake_quantile(plan, x, QS)
  src = _source(plan, x, np.float32)
  w = co.window_weights(plan.window_size)
  for h in range(plan.nhour):
    for d in range(int(plan.hour_nday[h])):
      win = _window(plan, src, h, d).astype(np.float64)
      wts = np.broadcast_to(w[:, None], win.shape[:2])
      for c in range(x.shape[1]):
        want = cq.weighted_quantile(win[..., c], wts, QS)
        _assert_float32_of(out[h, :, plan.out_row[h, d], c], want, (h, d, c))


@pytest.mark.parametrize('kw', [t[1] for t in TABLES], ids=[t[0] for t in
                                                             TABLES])
def test_fake_seeps_matches_the_oracle_window_by_window(kw):
  kw = dict(kw, kind='precip')
  plan, x = make_tables(6, **kw)
  thr_m = 0.25e-3  # not representable in float32: compared in x's precision
  x[::7] = x.dtype.type(thr_m)  # samples exactly at the threshold
  out, dry = fake_quantile(plan, x, [2 / 3], thr_m)
  src = _source(plan, x, np.float32)
  w = co.window_weights(plan.window_size)
  thr = src.dtype.type(thr_m)
  for h in range(plan.nhour):
    for d in range(int(plan.hour_nday[h])):
      win = _window(plan, src, h, d)
      wts = np.broadcast_to(w[:, None], win.shape[:2])
      r = plan.out_row[h, d]
      for c in range(x.shape[1]):
        if win.shape[1] == 0:  # no stacked year in this hour
          want = [np.nan, np.nan]
        else:
          want = cq.seeps_of_window(win[..., c], wts, thr)
        _assert_float32_of(np.array([out[h, 0, r, c], dry[h, r, c]]),
                           np.asarray(want, np.float64), (h, d, c))


def test_an_hour_without_items_gives_nan_quantiles_and_dry_fraction():
  plan, x = make_tables(7, nhour=2, nday=6, nitem=3, window_size=5,
                        kind='precip', absent_years={1: [0, 1, 2]})
  out, dry = fake_quantile(plan, x, [2 / 3], 0.25e-3)
  assert np.isnan(out[1]).all() and np.isnan(dry[1]).all()
  assert np.isfinite(dry[0]).all()


def test_generated_tables_have_the_requested_holes():
  plan, x = make_tables(8, nhour=3, nday=10, hour_nday=[1, 2, 10],
                        nday_out=12, nitem=4, absent_years={2: [1]},
                        missing=0.3, fill_missing=0.5, steps_per_day=2,
                        empty_days=0.3, nan_cells=(0,))
  for h in range(3):
    n = int(plan.hour_nday[h])
    rows = plan.out_row[h, :n]
    assert (np.diff(rows) > 0).all() and rows.max() < plan.nday_out
    assert (plan.items[h, n:] == -1).all()
  assert (plan.items[2, :, 1] == -1).all() and plan.fill[2, 1] == -1
  assert (plan.items == -1).any() and (plan.fill == -1).any()
  assert (plan.res_count == 0).any() and plan.nres == plan.items.size
  assert plan.items.max() < plan.nres and x.shape[0] == 2 * plan.nres
  assert np.isnan(x[:, 0]).all()

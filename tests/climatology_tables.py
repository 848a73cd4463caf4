"""TEST INFRASTRUCTURE: seeded index tables for the climatology entries of the
C ABI (wb2_climatology*, wb2_climatology_quantile*), at shapes and with holes
that `utils._plan` never produces from a time axis: short and uneven day axes,
missing items, absent stacked-year columns, missing fill steps, resampled days
without data, and fields with ties, zeros, a large offset or NaN.

`make_tables(...)` returns (plan, x): a `_lib.ClimatologyPlan` and the series
x [ntime][ncell] it indexes.  The tables are valid for the header: out_row is
increasing and injective within an hour, every step index is in range, and a
stacked year absent from an hour has no fill step either (as in the tables
`utils._plan` builds, where fill is the year's own day-365 step)."""
import numpy as np

from weatherbench2_b200 import _lib


def series(rs, shape, kind, dtype):
  """A field of the given kind: normal, offset (1e5 + 0.5 N), ties (values in
  {-0.0, 0.0, 0.5, 1.0}), constant (3.7) or precip (~40 % exact zeros)."""
  if kind == 'normal':
    x = rs.normal(size=shape)
  elif kind == 'offset':
    x = 1e5 + 0.5 * rs.normal(size=shape)
  elif kind == 'ties':
    x = np.array([-0.0, 0.0, 0.5, 1.0])[rs.randint(0, 4, size=shape)]
  elif kind == 'constant':
    x = np.full(shape, 3.7)
  elif kind == 'precip':
    x = np.where(rs.uniform(size=shape) < 0.4, 0.0,
                 rs.gamma(0.8, 2e-3, size=shape))
  else:
    raise ValueError(kind)
  return x.astype(dtype)


def make_tables(seed=0, *, nhour=1, nday=20, nitem=3, window_size=31,
                nday_out=None, method=0, dtype=np.float32, ncell=5,
                hour_nday=None, missing=0.0, empty_slots=0.0,
                absent_years=None, fill_missing=0.0, steps_per_day=0,
                empty_days=0.0, kind='normal', nan=0.0, nan_cells=()):
  """(plan, x).

  hour_nday     per-hour day slots (default nday for every hour)
  nday_out      output rows (default nday); out_row maps each hour's slots
                to an increasing random subset of them
  missing       fraction of items set to -1
  empty_slots   fraction of (hour, slot) whose every item is -1
  absent_years  {hour: [stacked-year column, ...]}: columns with no item and
                no fill step in that hour
  fill_missing  fraction of fill entries set to -1
  steps_per_day > 0: the tables index days of a daily resample (nres > 0),
                each the mean of that many consecutive steps of x; a fraction
                `empty_days` of the days has no step (res_count 0)
  kind, nan, nan_cells  the data (see `series`), a fraction of NaN values,
                and cells that are NaN everywhere
  """
  rs = np.random.RandomState(seed)
  hour_nday = np.asarray([nday] * nhour if hour_nday is None else hour_nday,
                         np.int32)
  assert hour_nday.shape == (nhour,) and hour_nday.max() <= nday
  nday_out = nday if nday_out is None else nday_out
  assert nday_out >= hour_nday.max()
  # every (hour, slot, year) item its own source step, scattered over time
  nsrc = nhour * nday * nitem
  items = rs.permutation(nsrc).reshape(nhour, nday, nitem).astype(np.int64)
  items[rs.uniform(size=items.shape) < missing] = -1
  items[rs.uniform(size=(nhour, nday)) < empty_slots] = -1
  fill = np.full((nhour, nitem), -1, np.int64)
  out_row = np.zeros((nhour, nday), np.int32)
  for h in range(nhour):
    n = int(hour_nday[h])
    items[h, n:] = -1  # slots past the hour's day axis are never read
    # the fill of year j: one of the year's own steps (its "day 365")
    fill[h] = items[h, rs.randint(0, n), :]
    out_row[h, :n] = np.sort(rs.choice(nday_out, n, replace=False))
  fill[rs.uniform(size=fill.shape) < fill_missing] = -1
  for h, cols in (absent_years or {}).items():
    items[h, :, cols] = -1
    fill[h, cols] = -1
  res_start = res_count = None
  if steps_per_day:
    assert dtype == np.float32, 'the daily resample takes float32 input'
    res_count = np.where(rs.uniform(size=nsrc) < empty_days, 0,
                         steps_per_day).astype(np.int32)
    res_start = (np.arange(nsrc) * steps_per_day).astype(np.int64)
    ntime = nsrc * steps_per_day
  else:
    ntime = nsrc
  x = series(rs, (ntime, ncell), kind, dtype)
  if nan:
    x[rs.uniform(size=x.shape) < nan] = np.nan
  x[:, list(nan_cells)] = np.nan
  plan = _lib.ClimatologyPlan(items, fill if method == 0 else None, hour_nday,
                              out_row, nday_out, window_size, method,
                              res_start, res_count)
  return plan, x

"""Reindexing datasets in time on the GPU: expanded climatologies, forecasts on
valid time, and probabilistic climatological forecasts.

Drop-ins for three of the reference's data-preparation scripts, without Beam
or zarr:

  expand_climatology        scripts/expand_climatology.py (`main` and
                            `select_climatology`)
  index_on_valid_time,      scripts/index_on_valid_time.py (`main` and
  get_forecast_offset_and_  `get_forecast_offset_and_spacing`)
  spacing
  compute_probabilistic_    scripts/compute_probabilistic_climatological_
  climatological_forecasts, forecasts.py (`main`, `_get_sampled_init_times`,
  get_sampled_init_times,   `_get_ensemble_size` and the flag checks)
  get_ensemble_size,
  sample_forecasts_core

Every output is one slab per outer index, copied from one source slab or
filled with NaN.  The plan is built on the host with NumPy from coordinates
and labels: per variable, one int64 offset table over the variable's own
strides (`_spatial.gather_operand` / `_spatial.offset_table`).  The slab is the
longest run of trailing dims that are not gathered and have the same order in
source and output, so no layout is copied and no dim order is refused.  The
copy is csrc/slab_gather.cu: CUDA data is read in place and gives CUDA
output; NumPy (np.memmap included) is streamed in bands within
`STREAM_BUDGET_BYTES`, and each band uploads only the source slabs it
references, so a forecast sampled from a long record reads a small part of it.
Datasets may be xarray or xarray_lite; the result is of the same kind.

Deviations from the reference:
- Data must be float32 or float64 (TypeError naming the variable), except
  that index_on_valid_time casts integer data to float64 on the host before
  the gather to float32.  For integers of magnitude above 2^53 that double
  rounding can differ by one float32 ulp from a direct cast to float32.
- A variable without the gathered dims raises ValueError naming it; the
  reference's pipelines cannot write such a variable either.
- A climatology with a single `hour` value raises ValueError; the reference
  raises IndexError.
- The reference raises `flags.ValidationError` in `_get_ensemble_size` and
  `_check_times_in_dataset`; these raise ValueError.
"""
from __future__ import annotations

import calendar
from typing import Optional, Sequence

import numpy as np
import pandas as pd

from weatherbench2_b200 import _lib
from weatherbench2_b200 import _spatial
from weatherbench2_b200 import _streamed
from weatherbench2_b200 import xarray_lite as xl

# device bytes of the two staging buffers of a NumPy source
STREAM_BUDGET_BYTES = 4 << 30

TIME = 'time'
DELTA = 'prediction_timedelta'
INIT = 'init'
REALIZATION = 'realization'
SOURCE_TIME = 'source_time'
VALID_AND_DELTA = 'valid_and_delta'
VALID_AND_INIT = 'valid_and_init'
WRAP_YEAR = 'WRAP_YEAR'
NO_EDGE = 'NO_EDGE'
REFLECT_RANGE = 'REFLECT_RANGE'
ONE_DAY = pd.Timedelta('1D')


def _source_dtype(da: xl.DataArray, allow_int: bool) -> np.dtype:
  """The dtype the gather reads `da` in: its own float32 / float64, or
  float64 for integers when `allow_int`."""
  dt = np.dtype(da.dtype) if not xl._is_torch(da.data) else np.dtype(  # pylint: disable=protected-access
      str(da.data.dtype).replace('torch.', ''))
  if dt in (np.float32, np.float64):
    return dt
  if allow_int and dt.kind in 'iu':
    return np.dtype(np.float64)
  raise TypeError(f'variable {da.name!r} has dtype {dt}: reindexing takes '
                  'float32 or float64 data'
                  + (' (or integers)' if allow_int else ''))


def _gather(da: xl.DataArray, out_dims: Sequence[str], out_sizes: dict,
            index_maps: dict, out_dtype, *, allow_int: bool = False):
  """out[...] = da indexed by `index_maps`, NaN where a position is -1.

  index_maps: {source dim: (output dims, int64 positions over them)}; every
  other dim of `da` appears in `out_dims` with the same size.  Returns the
  array of shape `out_sizes[d] for d in out_dims` (CUDA for CUDA data)."""
  src_dims, shape = tuple(da.dims), tuple(da.shape)
  gathered = set(index_maps) | {d for td, _ in index_maps.values() for d in td}
  k = 0
  while (k < min(len(src_dims), len(out_dims)) and
         src_dims[-1 - k] == out_dims[-1 - k] and src_dims[-1 - k] not in gathered):
    k += 1
  n_outer = len(src_dims) - k
  slab = int(np.prod(shape[n_outer:], dtype=np.int64))
  strides = [int(np.prod(shape[i + 1:], dtype=np.int64)) for i in range(n_outer)]
  src_elems = int(np.prod(shape, dtype=np.int64))
  src_dt = _source_dtype(da, allow_int)
  op = _spatial.Operand(
      data=None, addr=0, itemsize=src_dt.itemsize, on_device=False,
      outer_dims=src_dims[:n_outer], outer_shape=shape[:n_outer],
      outer_strides=tuple(strides), layout='lat_lon', nrow=1, ncol=slab,
      row_stride=slab, dtype=src_dt)
  odims = tuple(out_dims[:len(out_dims) - k])
  oshape = tuple(out_sizes[d] for d in odims)
  missing = np.zeros(oshape, bool)
  maps = {}
  for d, (tdims, pos) in index_maps.items():
    pos = np.asarray(pos, dtype=np.int64)
    bad = pos < 0
    if bad.any():
      perm = [tdims.index(x) for x in odims if x in tdims]
      m = np.transpose(bad, perm)[tuple(slice(None) if x in tdims else None
                                        for x in odims)]
      missing = missing | m
    maps[d] = (tuple(tdims), np.where(bad, 0, pos))
  table = np.where(missing.reshape(-1), -1, _spatial.offset_table(
      _spatial.gather_operand(op, maps), odims, oshape))
  oshape_full = tuple(out_sizes[d] for d in out_dims)
  out_dt = np.dtype(out_dtype)
  return _streamed.run(
      'slab_gather', da.data, (src_elems, slab, table.size, table),
      [(oshape_full, out_dt)], STREAM_BUDGET_BYTES, dtype=src_dt,
      out_dtype=_lib.F64 if out_dt == np.float64 else _lib.F32)[0]


def _positions(index: np.ndarray, labels, dim: str) -> np.ndarray:
  """Positions of `labels` in `index`; a missing label raises KeyError, as
  xarray's `sel` does."""
  pos = pd.Index(index).get_indexer(np.asarray(labels).reshape(-1))
  if (pos < 0).any():
    bad = np.asarray(labels).reshape(-1)[pos < 0]
    raise KeyError(f'not all values found in index {dim!r}: {bad[:10]}')
  return pos.reshape(np.shape(labels)).astype(np.int64)


def _other_coords(ds, drop_dims) -> dict:
  return {k: c for k, c in ds.coords.items()
          if not any(d in drop_dims for d in c.dims) and k not in drop_dims}


def _variables(ds, variables):
  if variables is None:
    return list(ds.keys())
  return [variables] if isinstance(variables, str) else list(variables)


# ---- expand_climatology ---------------------------------------------------------
@xl.boundary
def expand_climatology(climatology, *, time_start: str = '2017-01-01',
                       time_stop: str = '2017-12-31',
                       variables: Optional[Sequence[str]] = None):
  """scripts/expand_climatology.py without Beam or zarr: the climatology
  looked up by label (`sel(dayofyear=..., hour=...)`) at every time of
  `pd.date_range(time_start, time_stop, freq=hour_delta h)`, where hour_delta
  is hour[1] - hour[0], or 24 without an `hour` coordinate.  Output dims are
  (time, *other dims in source order); dayofyear and hour are dropped."""
  if 'hour' in climatology.coords:
    hours = np.asarray(climatology.coords['hour'].values)
    if hours.size < 2:
      raise ValueError('a climatology with an hour coordinate needs at least '
                       f'two hours to give the time step; it has {hours}')
    hour_delta = (hours[1] - hours[0]).item()
    time_dims = ('hour', 'dayofyear')
  else:
    hour_delta = 24
    time_dims = ('dayofyear',)
  times = pd.date_range(time_start, time_stop,
                        freq=hour_delta * pd.Timedelta('1h')).as_unit('ns')
  doy = climatology.coords['dayofyear'].values
  maps = {'dayofyear': ((TIME,), _positions(doy, times.dayofyear.values,
                                            'dayofyear'))}
  if 'hour' in time_dims:
    maps['hour'] = ((TIME,), _positions(hours, times.hour.values, 'hour'))
  coords = _other_coords(climatology, time_dims)
  coords[TIME] = xl.Coord((TIME,), times.values)
  out = xl.Dataset(coords=coords, attrs=climatology.attrs)
  for name in _variables(climatology, variables):
    da = climatology[name]
    lacking = [d for d in time_dims if d not in da.dims]
    if lacking:
      raise ValueError(f'variable {name!r} has no {lacking} dims to expand '
                       f'over time (dims {da.dims})')
    dims = (TIME,) + tuple(d for d in da.dims if d not in time_dims)
    sizes = dict(da.sizes, **{TIME: times.size})
    data = _gather(da, dims, sizes, maps, _source_dtype(da, False))
    out[name] = xl.DataArray(data, dims, name=name, attrs=da.attrs)
  return out


# ---- index_on_valid_time --------------------------------------------------------
def get_forecast_offset_and_spacing(init_times: np.ndarray,
                                    lead_times: np.ndarray) -> tuple[int, int]:
  """(offset, spacing) of the forecasts by valid time: the leads kept on valid
  time are lead_times[offset::spacing] (spacing = init step / lead step)."""
  init_times, lead_times = np.asarray(init_times), np.asarray(lead_times)
  init_steps = np.unique(np.diff(init_times))
  if init_steps.size > 1:
    raise ValueError(f'initialization times are not equidistant: {init_steps}')
  if init_steps.size == 0:
    raise ValueError('at least two initialization times are needed to find '
                     'their spacing')
  lead_steps = np.unique(np.diff(lead_times))
  if lead_steps.size > 1:
    raise ValueError(f'lead times are not equidistant: {lead_steps}')
  if lead_steps.size == 0:
    raise ValueError('at least two lead times are needed to find their spacing')
  init_delta, lead_delta = init_steps[0], lead_steps[0]
  spacing, remainder = divmod(init_delta, lead_delta)
  if remainder:
    raise ValueError(
        'initialization times not spaced at a multiple of lead times: '
        f'lead_delta={lead_delta!r}, init_delta={init_delta!r}')
  if lead_times[0] == np.timedelta64(0, 'h'):
    return 0, int(spacing)
  hits = np.flatnonzero(lead_times == spacing * lead_delta)
  if not hits.size:
    raise ValueError(f'{spacing * lead_delta!r} is not among the lead times')
  return int(hits[0]), int(spacing)


def _common_axis(ds, dim: str) -> int:
  axes = {}
  for name, da in ds.items():
    if dim not in da.dims:
      raise ValueError(f'variable {name!r} has no {dim!r} dim (dims {da.dims})')
    axes[name] = da.dims.index(dim)
  if len(set(axes.values())) > 1:
    raise ValueError(f'variables have {dim!r} at different axes: {axes}')
  return next(iter(axes.values()))


@xl.boundary
def index_on_valid_time(forecast, *,
                        desired_time_dims: str = VALID_AND_DELTA):
  """scripts/index_on_valid_time.py without Beam or zarr.  A
  (time=init, prediction_timedelta, ...) forecast on valid time `time` =
  unique(init + kept leads), float32, NaN where no forecast exists.

  valid_and_delta: leads offset::spacing are kept; `time` is valid time at the
  init axis's position.  valid_and_init: every lead is kept; the input `time`
  becomes `init` and valid `time` takes the lead axis's position."""
  if desired_time_dims not in (VALID_AND_DELTA, VALID_AND_INIT):
    raise ValueError(f'Unhandled desired_time_dims={desired_time_dims!r}')
  init = np.asarray(forecast.coords[TIME].values)
  leads = np.asarray(forecast.coords[DELTA].values)
  offset, spacing = get_forecast_offset_and_spacing(init, leads)
  _common_axis(forecast, TIME)
  _common_axis(forecast, DELTA)
  if desired_time_dims == VALID_AND_DELTA:
    kept = leads[offset::spacing]
    times = np.unique(init[:, None] + kept[None, :])
    init_pos = pd.Index(init).get_indexer(
        (times[:, None] - kept[None, :]).reshape(-1)).reshape(times.size,
                                                             kept.size)
    maps = {TIME: ((TIME, DELTA), init_pos),
            DELTA: ((DELTA,), offset + spacing * np.arange(kept.size))}
    rename = {TIME: TIME, DELTA: DELTA}
    sizes = {TIME: times.size, DELTA: kept.size}
    coords = {TIME: xl.Coord((TIME,), times), DELTA: xl.Coord((DELTA,), kept)}
  else:
    times = np.unique(init[:, None] + leads[None, :])
    lead_pos = pd.Index(leads).get_indexer(
        (times[None, :] - init[:, None]).reshape(-1)).reshape(init.size,
                                                             times.size)
    maps = {TIME: ((INIT,), np.arange(init.size)),
            DELTA: ((INIT, TIME), lead_pos)}
    rename = {TIME: INIT, DELTA: TIME}
    sizes = {INIT: init.size, TIME: times.size}
    coords = {INIT: xl.Coord((INIT,), init), TIME: xl.Coord((TIME,), times)}
  coords.update(_other_coords(forecast, (TIME, DELTA)))
  out = xl.Dataset(coords=coords, attrs=forecast.attrs)
  for name, da in forecast.items():
    dims = tuple(rename.get(d, d) for d in da.dims)
    data = _gather(da, dims, dict(da.sizes, **sizes), maps, np.float32,
                   allow_int=True)
    out[name] = xl.DataArray(data, dims, name=name, attrs=da.attrs)
  return out


# ---- probabilistic climatological forecasts ----------------------------------------
def _day_perturbations(day_window_size: int) -> np.ndarray:
  lo = (-day_window_size) // 2 + day_window_size % 2
  return np.arange(lo, lo + day_window_size)


def get_ensemble_size(ensemble_size: int, climatology_start_year: int,
                      climatology_end_year: int, day_window_size: int,
                      leave_out_if_in_climatology: bool) -> int:
  """The number of realizations: `ensemble_size`, or with -1 every (year, day
  perturbation) pair."""
  if ensemble_size == -1:
    if leave_out_if_in_climatology:
      raise ValueError(
          'ensemble_size=-1 (all combinations) is not supported when '
          'leave_out_if_in_climatology=True, as the number of available '
          'years can change per initial_time.')
    return (max(0, climatology_end_year - climatology_start_year + 1) *
            _day_perturbations(day_window_size).size)
  if ensemble_size > 0:
    return ensemble_size
  raise ValueError(
      f'ensemble_size={ensemble_size} but should be "-1" or a positive integer')


def _shuffled_rows(n_rows: int, n_times: int, n: int, seed: int) -> np.ndarray:
  """Row indices [n, n_times]: the first n of an independent random order of
  n_rows rows for every column, from a fresh generator seeded with `seed`."""
  order = np.random.default_rng(seed=seed).random((n_rows, n_times)).argsort(
      axis=0)
  if n < 1 or n > n_rows:
    raise ValueError(f'n must be None or in [1, x.shape[axis]] = [1, {n_rows}],'
                     f' found n={n}')
  return order[:n]


def _allowed_years(pool: np.ndarray, year: int, num_years_to_exclude: int):
  return [y for y in pool if y < year or y > year + num_years_to_exclude]


def get_sampled_init_times(
    output_times, *, climatology_start_year: int = 1990,
    climatology_end_year: int = 2020, day_window_size: int = 15,
    ensemble_size: int = 2, with_replacement: bool = True,
    sample_hold_days: int = 0, initial_time_edge_behavior: str = WRAP_YEAR,
    leave_out_if_in_climatology: bool = False, num_years_to_exclude: int = 0,
    seed: int = 802701) -> np.ndarray:
  """[ensemble_size, len(output_times)] datetime64[ns]: the truth time that
  starts realization i of the forecast initialised at output_times[j].

  A sampled time is year y, day of year output_time.dayofyear + delta and the
  output time's hour (minutes are dropped), with y drawn from
  [climatology_start_year, climatology_end_year] and delta from the
  day_window_size perturbations around 0; out-of-year days wrap within y
  (WRAP_YEAR), reflect at the first and last climatology year (REFLECT_RANGE)
  or cross into the next or previous year (NO_EDGE).  The draws come from
  `np.random.default_rng(seed)` in the order of the reference's
  `_get_sampled_init_times`, so the same arguments give the same times."""
  output_times = pd.DatetimeIndex(output_times).as_unit('ns')
  rng = np.random.default_rng(seed)
  if day_window_size <= 0 or day_window_size > 2 * 364:
    raise ValueError(
        f'day_window_size={day_window_size} not in [1, 2 * 364] but should be.')
  deltas = _day_perturbations(day_window_size)
  pool = np.arange(climatology_start_year, climatology_end_year + 1)
  n_times = len(output_times)
  if ensemble_size == -1:
    if leave_out_if_in_climatology:
      raise ValueError('ensemble_size=-1 (all combinations) is not supported '
                       'when leave_out_if_in_climatology=True.')
    ensemble_size = deltas.size * pool.size
  elif ensemble_size <= 0:
    raise ValueError(f'ensemble_size={ensemble_size} was not > 0 or -1.')
  shape = (ensemble_size, n_times)
  years = np.zeros(shape, dtype=int)
  lo, hi = deltas[0], deltas[-1] + 1

  if with_replacement:
    day_delta = rng.integers(lo, hi, size=shape)
    if not pool.size and ensemble_size > 0:
      raise ValueError(
          'Climatology year range is empty. Cannot sample years. Check '
          f'climatology_start_year={climatology_start_year}, '
          f'climatology_end_year={climatology_end_year}.')
    if leave_out_if_in_climatology:
      for j, t in enumerate(output_times):
        allowed = _allowed_years(pool, t.year, num_years_to_exclude)
        if not allowed:
          raise ValueError('No available climatology years to sample for '
                           'output_time')
        years[:, j] = rng.choice(allowed, size=ensemble_size, replace=True)
    elif pool.size:
      years = rng.integers(pool[0], pool[-1] + 1, size=shape)
  elif leave_out_if_in_climatology:
    for j, t in enumerate(output_times):
      allowed = _allowed_years(pool, t.year, num_years_to_exclude)
      if not allowed:
        raise ValueError('No available climatology years to sample for '
                         'output_time')
      if len(allowed) < ensemble_size:
        raise ValueError('Not enough available climatology years to sample '
                         'for output_time')
      years[:, j] = rng.choice(allowed, size=ensemble_size, replace=False)
      # drawn again for every output time; the last draw is the one used
      day_delta = rng.integers(lo, hi, size=shape)
  else:
    if not isinstance(seed, (int, np.integer)):
      raise ValueError(f'seed={seed!r} must be an integer to sample without '
                       'replacement')
    # every (year, perturbation) pair once per output time, in one random
    # order per column: row r is (pool[r // n_days], deltas[r % n_days])
    rows = _shuffled_rows(pool.size * deltas.size, n_times, ensemble_size,
                          seed)
    day_delta = deltas[rows % deltas.size]
    years = pool[rows // deltas.size]

  dayofyear = output_times.dayofyear.values + day_delta
  if initial_time_edge_behavior == WRAP_YEAR:
    for y in np.unique(years):
      m = years == y
      n_days = 365 + calendar.isleap(int(y))
      dayofyear[m] = (dayofyear[m] - 1) % n_days + 1
  elif initial_time_edge_behavior == REFLECT_RANGE:
    first = years == climatology_start_year
    dayofyear[first] = np.where(dayofyear[first] >= 1, dayofyear[first],
                                np.abs(dayofyear[first]) + 2)
    if climatology_end_year != climatology_start_year:
      last = years == climatology_end_year
      n_days = 365 + calendar.isleap(climatology_end_year)
      dayofyear[last] = np.where(dayofyear[last] <= n_days, dayofyear[last],
                                 2 * n_days - dayofyear[last])
  elif initial_time_edge_behavior != NO_EDGE:
    raise ValueError(
        f'Unhandled initial_time_edge_behavior={initial_time_edge_behavior!r}')

  sampled = (np.asarray(years - 1970, dtype='datetime64[Y]') +
             np.asarray(dayofyear - 1, dtype='timedelta64[D]') +
             np.asarray(output_times.hour, dtype='timedelta64[h]')).astype(
                 'datetime64[ns]')
  if sample_hold_days:
    strides = set(output_times.diff()[1:])
    if len(strides) > 1:
      raise ValueError(
          f'Cannot sample hold with more than one output_time_strides={strides}')
    stride = strides.pop()
    hold = pd.Timedelta(f'{sample_hold_days}D')
    hold_steps = hold // stride
    if stride * hold_steps != hold:
      raise ValueError(f'sample_hold_days={sample_hold_days} was not a '
                       f'multiple of output_time_stride={stride!r}')
    # whole days from each output time (floored), held for hold_steps times
    days = np.asarray(pd.to_timedelta(
        (sampled - output_times.values).ravel()).days, np.int64).reshape(shape)
    days = days[:, np.arange(n_times) // hold_steps]
    sampled = output_times.values + days.astype('timedelta64[D]')
  return sampled


def _check_time_spacing(times: np.ndarray, time_dim: str,
                        timedelta_spacing: str, initial_time_spacing: str):
  """The reference's `_check_input_spacing_and_time_flags`."""
  steps = np.unique(np.diff(times))
  if len(steps) != 1:
    raise ValueError(f'Non-unique spacing in INPUT along dim {time_dim}')
  input_step = pd.to_timedelta(steps[0])
  lead = pd.Timedelta(timedelta_spacing)
  init = pd.Timedelta(initial_time_spacing)
  if lead % init and init % lead:
    raise ValueError(
        f'Neither one of timedelta_spacing={timedelta_spacing!r} and '
        f'initial_time_spacing={initial_time_spacing!r} was a multiple of the '
        'other.')
  for name, value, step in (('TIMEDELTA_SPACING', timedelta_spacing, lead),
                            ('INITIAL_TIME_SPACING', initial_time_spacing,
                             init)):
    if step % input_step:
      raise ValueError(f'Requested {name}={value} is not a multiple of input '
                       f'spacing {input_step}')
    if step % ONE_DAY and ONE_DAY % step:
      raise ValueError(
          f'Requested {name}={value} was neither a multiple or divisor of one '
          'day. This will result in different times of day being used at '
          'different analysis points, which is inconvenient.')
    if step % pd.Timedelta('1h'):
      raise ValueError(f'Requested {name}={value} specified sub-hour '
                       'resolution.')


@xl.boundary
def sample_forecasts_core(truth, sampled_init_times, output_init_times,
                          timedeltas, *, realization_name: str = REALIZATION,
                          time_dim: str = TIME, add_source_time: bool = False,
                          missing_hint: str = ''):
  """Forecasts from truth: out[m, d, j] = truth at
  sampled_init_times[m, j] + timedeltas[d], dims (realization_name,
  prediction_timedelta, time_dim, *other dims in source order), the truth's
  dtype.  `sampled_init_times` [nmember, len(output_init_times)] may be any
  subset of a sampled table's columns with the matching output times.  With
  add_source_time, `source_time` (datetime64[ns]) holds the truth times read.
  A needed time the truth lacks raises ValueError listing the missing times."""
  sampled = np.asarray(sampled_init_times, dtype='datetime64[ns]')
  out_times = pd.DatetimeIndex(output_init_times).as_unit('ns')
  deltas = pd.TimedeltaIndex(timedeltas).as_unit('ns')
  if sampled.ndim != 2 or sampled.shape[1] != out_times.size:
    raise ValueError(f'sampled_init_times has shape {sampled.shape}; want '
                     f'(members, {out_times.size})')
  if DELTA in truth.sizes:
    raise ValueError(f'INPUT_PATH data already had {DELTA} as a dimension')
  needed = (sampled[:, None, :] +
            deltas.values.astype('timedelta64[ns]')[None, :, None])
  index = pd.Index(truth.coords[time_dim].values)
  missing = pd.to_datetime(np.unique(needed)).difference(index)
  if missing.size:
    raise ValueError(
        (missing_hint + '\n' if missing_hint else '') +
        'Time flags (INITIAL_TIME_EDGE_BEHAVIOR, CLIMATOLOGY_START_YEAR, '
        'CLIMATOLOGY_END_YEAR, TIMEDELTA_SPACING, SAMPLE_HOLD_DAYS) asked for '
        f'values in INPUT that are not available. missing_times={missing!r}.')
  pos = index.get_indexer(needed.reshape(-1)).reshape(needed.shape)
  head = (realization_name, DELTA, time_dim)
  sizes = {realization_name: sampled.shape[0], DELTA: deltas.size,
           time_dim: out_times.size}
  maps = {time_dim: (head, pos)}
  coords = _other_coords(truth, (time_dim,))
  coords.update({realization_name: xl.Coord((realization_name,),
                                            np.arange(sampled.shape[0])),
                 DELTA: xl.Coord((DELTA,), deltas.values),
                 time_dim: xl.Coord((time_dim,), out_times.values)})
  out = xl.Dataset(coords=coords, attrs=truth.attrs)
  for name, da in truth.items():
    if time_dim not in da.dims:
      raise ValueError(f'variable {name!r} has no {time_dim!r} dim to sample '
                       f'forecasts from (dims {da.dims})')
    dims = head + tuple(d for d in da.dims if d != time_dim)
    data = _gather(da, dims, dict(da.sizes, **sizes), maps,
                   _source_dtype(da, False))
    out[name] = xl.DataArray(data, dims, name=name, attrs=da.attrs)
  if add_source_time:
    out[SOURCE_TIME] = xl.DataArray(needed, head, name=SOURCE_TIME)
  return out


@xl.boundary
def compute_probabilistic_climatological_forecasts(
    truth, *, initial_time_start: str, initial_time_end: str,
    climatology_start_year: int = 1990, climatology_end_year: int = 2020,
    levels: Optional[Sequence] = None,
    variables: Optional[Sequence[str]] = None, time_dim: str = TIME,
    initial_time_spacing: str = '6h', sample_hold_days: int = 0,
    initial_time_edge_behavior: str = WRAP_YEAR,
    forecast_duration: str = '15 days', timedelta_spacing: str = '6h',
    add_source_time: bool = False, day_window_size: int = 15,
    ensemble_size: int = 2, with_replacement: bool = True,
    leave_out_if_in_climatology: bool = False, num_years_to_exclude: int = 0,
    seed: int = 802701, realization_name: str = REALIZATION):
  """scripts/compute_probabilistic_climatological_forecasts.py without Beam or
  zarr: for every init time of date_range(initial_time_start,
  initial_time_end, initial_time_spacing), ensemble_size stretches of truth of
  forecast_duration (leads every timedelta_spacing from 0), each starting at
  a time from `get_sampled_init_times`.  Keyword arguments are the script's
  flags, with its defaults."""
  if variables:
    truth = truth[[variables] if isinstance(variables, str)
                  else list(variables)]
  if levels:
    truth = truth.isel(level=_positions(truth.coords['level'].values,
                                        [int(l) for l in levels], 'level'))
  _check_time_spacing(np.asarray(truth.coords[time_dim].values), time_dim,
                      timedelta_spacing, initial_time_spacing)
  ensemble_size = get_ensemble_size(
      ensemble_size, climatology_start_year, climatology_end_year,
      day_window_size, leave_out_if_in_climatology)
  output_init_times = pd.date_range(initial_time_start, initial_time_end,
                                    freq=initial_time_spacing)
  timedeltas = pd.timedelta_range('0 days', forecast_duration,
                                  freq=timedelta_spacing)
  if DELTA in truth.sizes:
    raise ValueError(f'INPUT_PATH data already had {DELTA} as a dimension')
  sampled = get_sampled_init_times(
      output_init_times, climatology_start_year=climatology_start_year,
      climatology_end_year=climatology_end_year,
      day_window_size=day_window_size, ensemble_size=ensemble_size,
      with_replacement=with_replacement, sample_hold_days=sample_hold_days,
      initial_time_edge_behavior=initial_time_edge_behavior,
      leave_out_if_in_climatology=leave_out_if_in_climatology,
      num_years_to_exclude=num_years_to_exclude, seed=seed)
  hint = ''
  if initial_time_edge_behavior == WRAP_YEAR and sample_hold_days:
    hint = (f'initial_time_edge_behavior={initial_time_edge_behavior!r} and '
            f'sample_hold_days={sample_hold_days} means observations may be '
            'needed up to 1 year before/after the [CLIMATOLOGY_START_YEAR, '
            'CLIMATOLOGY_END_YEAR] interval.')
  return sample_forecasts_core(truth, sampled, output_init_times, timedeltas,
                               realization_name=realization_name,
                               time_dim=time_dim,
                               add_source_time=add_source_time,
                               missing_hint=hint)

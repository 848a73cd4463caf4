"""Per-chunk evaluation loop -- the API surface of weatherbench2/evaluation.py
that sits directly on the metric kernels:

  _metric_and_region_loop   (evaluation.py:388-438)
  _evaluate_all_metrics     (evaluation.py:441-483)
  evaluate_in_memory        (evaluation.py:486-517)

The reference loops metric x region in Python and every iteration re-reads the
chunk; here the loop runs inside `metrics.batch(...)`, so the first metric of a
family launches ONE kernel pass for all regions (and shares it with ACC's
climatology pass) and the remaining iterations only slice the result.

Zarr / netCDF I/O and the Beam pipeline (evaluation.py:520-828) are out of
scope (SURVEY.md section 8): datasets are passed in memory through
`config.Paths`; results are returned and saved as `.npz`.
"""
from __future__ import annotations

import copy
import dataclasses
import logging
import os
import typing as t

import numpy as np
import pandas as pd

from weatherbench2_b200 import config
from weatherbench2_b200 import metrics as metrics_lib
from weatherbench2_b200 import xarray_lite as xl


def make_latitude_increasing(dataset: xl.Dataset) -> xl.Dataset:
  """Flip the dataset if latitude is decreasing (evaluation.py:40-46)."""
  lat = dataset['latitude'].values
  if (np.diff(lat) < 0).all():
    dataset = dataset.isel(latitude=np.arange(lat.size)[::-1])
  return dataset


def apply_time_conventions(forecast: xl.Dataset, by_init: bool) -> xl.Dataset:
  """WeatherBench2 time names on a forecast (weatherbench2/schema.py:25-44)."""
  if 'prediction_timedelta' in forecast.coords:
    forecast = forecast.rename({'prediction_timedelta': 'lead_time'})
    if by_init:
      forecast = forecast.rename({'time': 'init_time'})
      init = forecast['init_time']
      lead = forecast['lead_time']
      valid = init.values[:, None] + lead.values[None, :]
      forecast = forecast.assign_coords(
          valid_time=(('init_time', 'lead_time'), valid))
    else:
      t_ = forecast['time']
      lead = forecast['lead_time']
      forecast = forecast.assign_coords(
          init_time=(('time', 'lead_time'),
                     t_.values[:, None] - lead.values[None, :]))
  return forecast


def select_truth_at_valid_time(truth: xl.Dataset, forecast: xl.Dataset
                               ) -> xl.Dataset:
  """`truth.sel(time=forecast.valid_time)` (evaluation.py:475) WITHOUT
  materialising the (init_time, lead_time, ...) copy: each variable becomes a
  LazyGather view whose label lookup is folded into the kernels' offset table.
  """
  vt = forecast['valid_time']
  # like xarray's sel with a DataArray indexer, the result carries the
  # indexer's coordinates (init_time and lead_time, which derived variables
  # along lead time read)
  extra = {k: c for k, c in forecast.coords.items()
           if c.dims and all(d in vt.dims for d in c.dims)}
  extra['valid_time'] = xl.Coord(vt.dims, vt.values)
  out = xl.Dataset(attrs=truth.attrs)
  for k in truth.keys():
    v = truth[k]
    if 'time' not in v.dims:
      out[k] = v
      continue
    pos = xl._lookup(v.coords['time'].values, vt.values.ravel())  # pylint: disable=protected-access
    out[k] = LazyGather(v, {'time': (vt.dims, pos.reshape(vt.shape))},
                        extra_coords=extra)
  return out


LazyGather = xl.LazyGather  # defined next to the container it extends


@xl.boundary
def _metric_and_region_loop(forecast: xl.Dataset, truth: xl.Dataset,
                            eval_config: config.Eval, skipna: bool,
                            compute_chunk: bool = False) -> xl.Dataset:
  """Metric results looping over metrics and regions (evaluation.py:388-438).
  Result variables have dims (metric, [region], ...)."""
  logging.info('Starting _metric_and_region_loop')
  for name, dv in eval_config.derived_variables.items():
    forecast[name] = dv.compute(forecast)
    truth[name] = dv.compute(truth)

  regions = (list(eval_config.regions.values())
             if eval_config.regions is not None else [None])
  climatology = None
  for metric in eval_config.metrics.values():
    if isinstance(metric, metrics_lib.ACC):
      climatology = xl.from_xarray(metric.climatology)
      break

  results = []
  with metrics_lib.batch(regions, climatology):
    for name, metric in eval_config.metrics.items():
      logging.info('Logging metric: %s', name)
      if compute_chunk or not eval_config.temporal_mean:
        eval_fn = metric.compute_chunk
      else:
        eval_fn = metric.compute
      if eval_config.regions is not None:
        tmp_results = []
        for region_name, region in eval_config.regions.items():
          tmp = eval_fn(forecast=forecast, truth=truth, region=region,
                        skipna=skipna)
          tmp_results.append(tmp.expand_dims(
              {'metric': np.array([name], dtype=object),
               'region': np.array([region_name], dtype=object)}))
        result = xl.concat(tmp_results, 'region')
      else:
        result = eval_fn(forecast=forecast, truth=truth,
                         skipna=skipna).expand_dims(
                             {'metric': np.array([name], dtype=object)})
      results.append(result)
  return xl.merge(results)


def _ensure_nonempty(dataset: xl.Dataset, message: str = '') -> None:
  """evaluation.py:65-68."""
  sizes = dataset.sizes
  if sizes and not min(sizes.values()):
    raise ValueError(f'`dataset` was empty: {sizes=}.  {message}')


def _decode_pressure_level_suffixes(forecast: xl.Dataset) -> xl.Dataset:
  """Variables stored as `<name>_<level>` become `<name>` with a `level`
  dimension (evaluation.py:71-89); levels of one name are stacked in
  ascending order (the outer join of `xr.merge` sorts the labels)."""
  if 'channel' in forecast.sizes and 'forecast' in forecast.keys():
    da = forecast['forecast']
    forecast = xl.Dataset(
        {str(c): da.isel(channel=i, drop=True)
         for i, c in enumerate(da.coords['channel'].values)}, attrs=forecast.attrs)
  plain, by_name = {}, {}
  for var in forecast.keys():
    name, _, suffix = str(var).rpartition('_')
    if name and suffix.isdigit():
      by_name.setdefault(name, []).append((int(suffix), forecast[var]))
    else:
      plain[str(var)] = forecast[var]
  out = xl.Dataset(attrs=forecast.attrs)
  for name, da in plain.items():
    out[name] = da
  for name, members in by_name.items():
    members.sort(key=lambda m: m[0])
    first = members[0][1]
    data = np.stack([np.asarray(m[1].values) for m in members])
    coords = dict(first.coords)
    coords['level'] = xl.Coord(('level',), np.array([m[0] for m in members]))
    out[name] = xl.DataArray(data, ('level',) + first.dims, coords, name,
                             first.attrs)
  return out


def _impose_data_selection(dataset: xl.Dataset, selection: config.Selection,
                           select_time: bool = True,
                           time_dim: t.Optional[str] = None,
                           select_aux: bool = False,
                           optional: t.Collection[str] = ()) -> xl.Dataset:
  """Variables, latitude / longitude box, levels and time range of a
  config.Selection (evaluation.py:139-162).  `optional` names (derived
  variables, computed later from their base variables) may be absent."""
  names = list(selection.variables)
  if select_aux and selection.aux_variables is not None:
    names += [v for v in selection.aux_variables if v not in names]
  names = [v for v in names if v in dataset.keys() or v not in optional]
  dataset = dataset[names]  # KeyError for a missing variable, like xarray
  box = {}
  for dim, sl in (('latitude', selection.lat_slice),
                  ('longitude', selection.lon_slice)):
    if sl is not None and sl != slice(None, None) and dim in dataset.sizes:
      box[dim] = sl
  if box:
    dataset = dataset.sel(box)
  if selection.levels is not None and 'level' in dataset.sizes:
    dataset = dataset.sel(level=np.asarray(selection.levels))
  if select_time and selection.time_slice is not None and (
      selection.time_slice != slice(None, None)):
    dataset = dataset.sel({time_dim: _as_datetime_slice(selection.time_slice)})
  _ensure_nonempty(dataset, 'Selection created empty dataset')
  return dataset


def create_persistence_forecast(forecast: xl.Dataset, obs: xl.Dataset
                                ) -> xl.Dataset:
  """Observation at the forecast's initialisation time, shaped like the
  forecast -- as lazily gathered views of `obs`, no copy.

  By-valid forecasts (dims time, lead_time; 2-D `init_time` coordinate) follow
  evaluation.py:165-193: valid times before `time[0] + max(lead_time)` are
  dropped.  By-init forecasts follow the reference's Beam path
  (evaluation.py:644-656): `truth.sel(time=init_time)` repeated along
  `lead_time`, with the forecast's `valid_time` coordinate."""
  if 'init_time' in forecast.sizes:  # by-init
    init = forecast.coords['init_time'].values
    lead = forecast.coords['lead_time'].values
    tdims = ('init_time', 'lead_time')
    labels = np.broadcast_to(init[:, None], (init.size, lead.size))
    extra = {'init_time': xl.Coord(('init_time',), init),
             'lead_time': xl.Coord(('lead_time',), lead),
             'valid_time': xl.Coord(tdims, init[:, None] + lead[None, :])}
  else:
    logging.warning('by-valid with evaluate_persistence is not 100% correct.')
    it = forecast['init_time']  # (time, lead_time) in some order
    times = forecast.coords['time'].values
    lead = forecast.coords['lead_time'].values
    keep = xl.label_slice_indices(times, slice(times[0] + lead.max(), None))
    it = it.isel(time=keep)
    tdims = it.dims
    labels = it.values
    extra = {'time': xl.Coord(('time',), times[keep]),
             'lead_time': xl.Coord(('lead_time',), lead)}
  out = xl.Dataset(attrs=obs.attrs)
  for k in obs.keys():
    v = obs[k]
    if 'time' not in v.dims:
      out[k] = v
      continue
    pos = xl._lookup(v.coords['time'].values, labels.ravel())  # pylint: disable=protected-access
    out[k] = LazyGather(v, {'time': (tdims, pos.reshape(labels.shape))},
                        extra_coords=extra)
  return out


def climatology_forecast(climatology: xl.Dataset, forecast: xl.Dataset,
                         time_dim: str) -> xl.Dataset:
  """`climatology[list(forecast)].sel(dayofyear=..., hour=...)` at the
  forecast's (valid) times (evaluation.py:452-457, 467-471) -- as lazily
  gathered views: the kernels read the climatology slabs in place through the
  offset table instead of a forecast-sized copy.  Like the reference's Beam
  path (evaluation.py:620-638) a climatology without `hour` is looked up by day
  of year only and `<name>_mean` variables stand in for `<name>`."""
  names = [str(k) for k in forecast.keys()]
  try:
    clim = climatology[names]
  except KeyError:
    renames = {k + '_mean': k for k in names}
    clim = climatology[list(renames)].rename(renames)
  vt = forecast[time_dim]
  stamps = pd.DatetimeIndex(np.asarray(vt.values).ravel())
  doy = np.asarray(stamps.dayofyear).reshape(vt.shape)
  hour = np.asarray(stamps.hour).reshape(vt.shape)
  extra = {k: c for k, c in vt.coords.items()}
  extra[time_dim] = xl.Coord(vt.dims, vt.values)
  extra['dayofyear'] = xl.Coord(vt.dims, doy)
  out = xl.Dataset(attrs=climatology.attrs)
  for k in names:
    v = clim[k]
    if 'level' in v.dims and 'level' in forecast.coords:
      # the later arithmetic joins levels by label anyway (inner join)
      have = v.coords['level'].values
      want = forecast.coords['level'].values
      want = want[np.isin(want, have)]
      if want.size != have.size or (want != have).any():
        v = v.sel(level=want)
    maps = {'dayofyear': (vt.dims, xl._lookup(  # pylint: disable=protected-access
        v.coords['dayofyear'].values, doy.ravel()).reshape(vt.shape))}
    coords = dict(extra)
    if 'hour' in v.dims:
      maps['hour'] = (vt.dims, xl._lookup(  # pylint: disable=protected-access
          v.coords['hour'].values, hour.ravel()).reshape(vt.shape))
      coords['hour'] = xl.Coord(vt.dims, hour)
    out[k] = LazyGather(v, maps, extra_coords=coords)
  return out


def make_probabilistic_climatology(ds: xl.Dataset, start_year: int,
                                   end_year: int, hour_interval: int
                                   ) -> xl.Dataset:
  """Years of the ground truth stacked as ensemble members
  (weatherbench2/utils.py:47-70): dims (hour, number, dayofyear, ...); day 366
  holds data for leap years only (NaN elsewhere), as do days a year lacks."""
  times = pd.DatetimeIndex(ds.coords['time'].values)
  hours = np.arange(0, 24, hour_interval)
  years = np.arange(start_year, end_year + 1)
  in_years = (times.year >= start_year) & (times.year <= end_year)
  days = np.unique(np.asarray(times.dayofyear)[
      in_years & np.isin(times.hour, hours)])
  if not days.size:
    raise ValueError('no ground truth inside the climatology years / hours')
  day_pos = {int(d): i for i, d in enumerate(days)}
  out = xl.Dataset(attrs=ds.attrs)
  for k in ds.keys():
    v = ds[k]
    if 'time' not in v.dims:
      continue
    src = np.moveaxis(np.asarray(v.values), v.dims.index('time'), 0)
    dtype = src.dtype if src.dtype.kind == 'f' else np.float64
    data = np.full((hours.size, years.size, days.size) + src.shape[1:], np.nan,
                   dtype=dtype)
    for hi, hour in enumerate(hours):
      for yi, year in enumerate(years):
        sel = np.nonzero((times.hour == hour) & (times.year == year))[0]
        if not sel.size:
          continue
        dpos = np.array([day_pos[int(d)] for d in times.dayofyear[sel]])
        if np.unique(dpos).size != dpos.size:
          raise ValueError(f'more than one time per day at hour {hour}')
        data[hi, yi, dpos] = src[sel]
    dims = ('hour', 'number', 'dayofyear') + tuple(
        d for d in v.dims if d != 'time')
    coords = {c: cc for c, cc in v.coords.items() if 'time' not in cc.dims}
    coords.update(hour=xl.Coord(('hour',), hours),
                  number=xl.Coord(('number',), np.arange(years.size)),
                  dayofyear=xl.Coord(('dayofyear',), days))
    out[k] = xl.DataArray(data, dims, coords, k, v.attrs)
  return out


def _unique_step_size(data: np.ndarray):
  """evaluation.py:196-205."""
  data = np.asarray(data)
  if data.ndim != 1:
    raise ValueError(f'array has wrong number of dimensions: {data.ndim}')
  if len(data) < 2:
    raise ValueError(f'{len(data)=}, which is too small to determine step size')
  uniques = np.unique(np.diff(data))
  if uniques.size != 1:
    raise ValueError(f'too many unique values: {uniques}')
  return uniques[0]


def _ensure_consistent_time_step_sizes(truth: xl.Dataset, forecast: xl.Dataset):
  """By-valid data: thin the finer of the two time axes
  (evaluation.py:208-230)."""
  truth_step = _unique_step_size(truth.coords['time'].values)
  forecast_step = _unique_step_size(forecast.coords['time'].values)
  if truth_step > forecast_step:
    multiple, remainder = divmod(truth_step, forecast_step)
    if remainder:
      raise ValueError('truth time step not a multiple of forecast time step: '
                       f'{truth_step} vs {forecast_step}')
    forecast = forecast.isel(time=slice(None, None, int(multiple)))
  elif truth_step < forecast_step:
    multiple, remainder = divmod(forecast_step, truth_step)
    if remainder:
      raise ValueError('forecast time step not a multiple of truth time step: '
                       f'{forecast_step} vs {truth_step}')
    truth = truth.isel(time=slice(None, None, int(multiple)))
  return truth, forecast


def _add_base_variables(data_config: config.Data, eval_config: config.Eval
                        ) -> config.Data:
  """Selection extended by the base variables of the derived variables
  (evaluation.py:233-256).  The datasets themselves are shared, not copied."""
  selection = copy.copy(data_config.selection)
  names = list(selection.variables)
  for dv in eval_config.derived_variables.values():
    names += [v for v in dv.base_variables if v not in names]
  selection.variables = names
  return dataclasses.replace(data_config, selection=selection)


def _select_analysis_init_time(forecast: xl.Dataset,
                               forecast_all_times: xl.Dataset):
  """Forecast / analysis pairing for by-init data evaluated against its own
  lead-0 fields (evaluation.py:259-293)."""
  analysis = forecast_all_times.sel(lead_time=np.timedelta64(0, 'ns'),
                                    drop=True)
  analysis = analysis.drop_vars(['valid_time']).rename({'init_time': 'time'})
  init_interval = np.diff(analysis.coords['time'].values)
  if not (init_interval == init_interval[0]).all():
    raise ValueError(f'Not all init_time intervals are equal: {init_interval}')
  init_interval = init_interval[0]
  lead_interval = np.diff(forecast.coords['lead_time'].values)
  assert np.all(lead_interval == lead_interval[0]), (
      'Not all lead_time intervals are equal.')
  lead_interval = lead_interval[0]
  assert init_interval >= lead_interval, (
      'Initialization interval cannot be less that lead_time interval.')
  lead_per_init = float(init_interval / lead_interval)
  assert lead_per_init.is_integer(), 'Init must be multiple of lead.'
  assert (analysis.coords['time'].values.max() >=
          forecast.coords['valid_time'].values.max()), (
              'Analysis does not extend to latest forecast init+lead')
  forecast = forecast.isel(lead_time=slice(None, None, int(lead_per_init)))
  return forecast, analysis


def open_forecast_and_truth_datasets(data_config: config.Data,
                                     eval_config: config.Eval):
  """In-memory restatement of evaluation.py:92-136, 296-365 for datasets passed
  through `config.Paths`: pressure-level suffixes, renames, latitude
  orientation, grid alignment, time conventions, the config.Selection
  (variables + base variables of derived ones, lat / lon box, levels, time
  range), the analysis-as-truth pairing and by-valid step thinning.  Zarr
  paths need xarray + zarr."""
  def _open(obj, what):
    if obj is None:
      return None
    if isinstance(obj, (str, os.PathLike)):
      if not xl.have_xarray():
        raise RuntimeError(
            f'{what}: zarr paths need xarray + zarr, which are not installed; '
            'pass an in-memory dataset in config.Paths instead')
      import xarray as xr  # pylint: disable=import-outside-toplevel
      return xl.from_xarray(xr.open_zarr(obj))
    return xl.from_xarray(obj)

  derived = set(eval_config.derived_variables)
  data_config = _add_base_variables(data_config, eval_config)
  sel = data_config.selection
  forecast = _open(data_config.paths.forecast, 'forecast')
  obs = _open(data_config.paths.obs, 'obs')
  climatology = _open(data_config.paths.climatology, 'climatology')
  if data_config.pressure_level_suffixes:
    forecast = _decode_pressure_level_suffixes(forecast)
  if data_config.rename_variables is not None:
    forecast = forecast.rename(data_config.rename_variables)
  obs = make_latitude_increasing(obs)
  forecast = make_latitude_increasing(forecast)
  if climatology is not None:
    climatology = make_latitude_increasing(climatology)
  for coord_name in ('latitude', 'longitude'):  # evaluation.py:49-61
    np.testing.assert_allclose(forecast[coord_name].values,
                               obs[coord_name].values, atol=1e-3)
  # _ensure_aligned_grid (evaluation.py:49-61): after the closeness check ONE
  # set of coordinates replaces the others', so that float32 / float64
  # coordinate labels cannot turn the later label joins into gathers
  grid = {k: forecast[k].values for k in ('latitude', 'longitude')}
  obs = obs.assign_coords(grid)
  if climatology is not None:
    for coord_name in ('latitude', 'longitude'):
      np.testing.assert_allclose(forecast[coord_name].values,
                                 climatology[coord_name].values, atol=1e-3)
    climatology = climatology.assign_coords(grid)
    box = {d: s for d, s in (('latitude', sel.lat_slice),
                             ('longitude', sel.lon_slice))
           if s is not None and s != slice(None, None)}
    if box:
      climatology = climatology.sel(box)
  forecast = apply_time_conventions(forecast, data_config.by_init)
  _ensure_nonempty(obs)
  _ensure_nonempty(forecast)

  time_dim = 'init_time' if data_config.by_init else 'time'
  forecast_all_times = None
  if eval_config.against_analysis and data_config.by_init:
    forecast_all_times = _impose_data_selection(
        forecast, sel, select_time=False, select_aux=True, optional=derived)
  if data_config.by_init:  # the matching truth times are gathered later
    obs = _impose_data_selection(obs, sel, select_time=False, optional=derived)
  else:
    obs = _impose_data_selection(obs, sel, time_dim='time', optional=derived)
  forecast = _impose_data_selection(forecast, sel, time_dim=time_dim,
                                    select_aux=True, optional=derived)
  if eval_config.against_analysis:
    eval_truth = forecast.sel(lead_time=np.timedelta64(0, 'ns'), drop=True)
    if data_config.by_init:
      forecast, eval_truth = _select_analysis_init_time(forecast,
                                                        forecast_all_times)
  else:
    eval_truth = obs
  if not data_config.by_init:
    eval_truth, forecast = _ensure_consistent_time_step_sizes(eval_truth,
                                                              forecast)
  return forecast, eval_truth, climatology


def _as_datetime_slice(s: slice) -> slice:
  """Label slice with datetime64 bounds.  String bounds follow pandas' partial
  string indexing, which xarray's `.sel(time=slice('2020-01-01', '2020-12-31'))`
  uses: a bound covers its whole period, so the stop '2020-12-31' includes
  every time of that day and '2020' the whole year."""
  def cv(x, end):
    if x is None:
      return None
    if isinstance(x, str):
      period = pd.Period(x)
      stamp = period.end_time if end else period.start_time
      return np.datetime64(stamp.value, 'ns')
    return np.datetime64(x, 'ns')
  return slice(cv(s.start, False), cv(s.stop, True))


def _get_output_path(data_config: config.Data, eval_name: str, fmt: str) -> str:
  # evaluation.py:368-380
  suffix = {'netcdf': 'nc', 'zarr': 'zarr', 'npz': 'npz'}[fmt]
  return os.path.join(
      data_config.paths.output_dir,
      f'{data_config.paths.output_file_prefix}{eval_name}.{suffix}')


def save_results(results: xl.Dataset, path: str) -> None:
  """netCDF when xarray is importable (evaluation.py:383-385), else .npz
  holding every variable, its dims and the coordinates."""
  if xl.have_xarray() and path.endswith('.nc'):
    xl.to_xarray(results).to_netcdf(path)
    return
  if xl.have_xarray() and path.endswith('.zarr'):
    xl.to_xarray(results).to_zarr(path)
    return
  payload = {}
  for k in results.keys():
    payload[f'var:{k}'] = results[k].values
    payload[f'dims:{k}'] = np.array(results[k].dims, dtype=object)
  for k, c in results.coords.items():
    payload[f'coord:{k}'] = c.values
    payload[f'coorddims:{k}'] = np.array(c.dims, dtype=object)
  os.makedirs(os.path.dirname(path) or '.', exist_ok=True)
  np.savez(path, **payload, allow_pickle=True)


def _baseline_forecast(forecast: xl.Dataset, truth: xl.Dataset, climatology,
                       eval_config: config.Eval, by_init: bool) -> xl.Dataset:
  """The forecast config.Eval asks to evaluate (evaluation.py:450-472): the
  model forecast itself, or a climatological / probabilistic-climatological /
  persistence forecast of the same shape -- as lazily gathered views (the
  reference materialises each with `.sel`): the kernels address the
  climatology / observation slabs in place."""
  time_dim = 'valid_time' if by_init else 'time'
  if eval_config.evaluate_climatology:
    if climatology is None:
      raise ValueError('evaluate_climatology needs config.Paths.climatology')
    forecast = climatology_forecast(climatology, forecast, time_dim)
  if eval_config.evaluate_probabilistic_climatology:
    probabilistic_climatology = make_probabilistic_climatology(
        truth, eval_config.probabilistic_climatology_start_year,
        eval_config.probabilistic_climatology_end_year,
        eval_config.probabilistic_climatology_hour_interval)
    forecast = climatology_forecast(probabilistic_climatology, forecast,
                                    time_dim)
  if eval_config.evaluate_persistence:
    forecast = create_persistence_forecast(forecast, truth)
  return forecast


def _save(results: xl.Dataset, data_config: config.Data, eval_name: str,
          eval_config: config.Eval) -> None:
  fmt = eval_config.output_format if xl.have_xarray() else 'npz'
  output_path = _get_output_path(data_config, eval_name, fmt)
  save_results(results, output_path)
  logging.info('Logging Saved results to %s', output_path)


def _evaluate_all_metrics(eval_name: str, eval_config: config.Eval,
                          data_config: config.Data, skipna: bool):
  """Evaluate a set of eval metrics in memory (evaluation.py:441-483)."""
  forecast, truth, climatology = open_forecast_and_truth_datasets(
      data_config, eval_config)
  forecast = _baseline_forecast(forecast, truth, climatology, eval_config,
                                data_config.by_init)
  if data_config.by_init:
    truth = select_truth_at_valid_time(truth, forecast)  # evaluation.py:475
  results = _metric_and_region_loop(forecast, truth, eval_config,
                                    skipna=skipna)
  _save(results, data_config, eval_name, eval_config)
  return results


def evaluate_in_memory(data_config: config.Data,
                       eval_configs: dict, skipna: bool = False) -> dict:
  """Run evaluation in memory, one results file per config.Eval
  (evaluation.py:486-517).  Also returns {eval_name: results}."""
  out = {}
  for eval_name, eval_config in eval_configs.items():
    out[eval_name] = _evaluate_all_metrics(eval_name, eval_config, data_config,
                                           skipna=skipna)
  return out


def evaluate_distributed(data_config: config.Data, eval_configs: dict, *,
                         input_chunks: t.Optional[t.Mapping[str, int]] = None,
                         num_threads: t.Optional[int] = None,
                         skipna: bool = False, prefetch: int = 2, group=None,
                         device=None) -> dict:
  """The chunked, multi-GPU evaluation: what `evaluate_with_beam` is to the
  reference (evaluation.py:556-828), on a `torch.distributed` process group
  with one process per GPU.

  For every config.Eval the datasets are opened and the baseline forecast is
  set up exactly as in `_evaluate_all_metrics`; chunks of
  `input_chunks['init_time']` (by-init) or `input_chunks['time']` (by-valid)
  time steps are sharded over the ranks (distributed.evaluate_sharded: pinned
  chunk feeder with `num_threads` readers, slab cache, one all-reduce of
  [sum, count] for the temporal mean -- or a gather of the per-chunk results
  when `temporal_mean=False`).  Other entries of `input_chunks` (lead_time,
  level, ...) are ignored: a chunk always holds all leads / levels, which the
  kernels take in one launch.  Every rank returns {eval_name: results}; rank
  0 writes the result files.  Without a process group it runs on one GPU.
  """
  from weatherbench2_b200 import distributed  # pylint: disable=import-outside-toplevel
  chunk_dim = 'init_time' if data_config.by_init else 'time'
  chunk_size = int((input_chunks or {}).get(chunk_dim, 1))
  if chunk_size < 1:  # xarray-beam's -1 = "the whole dimension in one chunk"
    chunk_size = None
  import torch.distributed as dist  # pylint: disable=import-outside-toplevel
  rank = dist.get_rank(group) if (dist.is_available() and
                                  dist.is_initialized()) else 0
  out = {}
  for eval_name, eval_config in eval_configs.items():
    forecast, truth, climatology = open_forecast_and_truth_datasets(
        data_config, eval_config)
    forecast = _baseline_forecast(forecast, truth, climatology, eval_config,
                                  data_config.by_init)
    baseline = (eval_config.evaluate_climatology or
                eval_config.evaluate_probabilistic_climatology or
                eval_config.evaluate_persistence)
    results = distributed.evaluate_sharded(
        forecast, truth, eval_config, skipna=skipna, chunk_dim=chunk_dim,
        chunk_size=chunk_size or forecast.sizes[chunk_dim], group=group,
        device=device,
        # a baseline forecast is a view of resident climatology / observation
        # slabs: nothing to read ahead (a feeder would copy it chunk by chunk)
        prefetch=0 if baseline else prefetch, num_threads=num_threads or 2,
        temporal_mean=bool(eval_config.temporal_mean))
    if rank == 0:
      _save(results, data_config, eval_name, eval_config)
    out[eval_name] = results
  return out


def evaluate_with_beam(data_config: config.Data, eval_configs: dict, *,
                       input_chunks: t.Mapping[str, int],
                       runner: t.Optional[str] = None,
                       fanout: t.Optional[int] = None,
                       shuffle_before_temporal_mean: bool = False,
                       num_threads: t.Optional[int] = None,
                       argv: t.Optional[list] = None,
                       skipna: bool = False) -> dict:
  """Drop-in for callers of the reference's `evaluate_with_beam`
  (evaluation.py:758-828; `scripts/evaluate.py`): same arguments, same result
  files, run by `evaluate_distributed`.  `runner`, `fanout`, `argv` and
  `shuffle_before_temporal_mean` steer the Beam runner and have no meaning
  here; they are accepted and ignored."""
  del runner, fanout, shuffle_before_temporal_mean, argv
  return evaluate_distributed(data_config, eval_configs,
                              input_chunks=input_chunks,
                              num_threads=num_threads, skipna=skipna)

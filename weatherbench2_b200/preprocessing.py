"""Device-side preprocessing that feeds the metric kernels (SURVEY.md section 8
f3): the ensemble mean of scripts/compute_ensemble_mean.py:110-141
(`xbeam.Mean(realization, skipna)`) computed in HBM, so that ensemble-mean
RMSE / ACC through K1 need no host round trip of the mean; the quantiles
of scripts/compute_quantiles.py (`Dataset.quantile` over chosen dims,
csrc/quantile.cu); and the area-weighted averages and raw moments of
scripts/compute_averages.py and compute_statistical_moments.py
(csrc/average.cu)."""
from __future__ import annotations

import math
from typing import Optional, Sequence

import numpy as np
import pandas as pd

from weatherbench2_b200 import _lib
from weatherbench2_b200 import _streamed
from weatherbench2_b200 import xarray_lite as xl

REALIZATION = 'realization'
QUANTILE = 'quantile'
# device bytes of the two staging buffers of a host (NumPy) quantile call
QUANTILE_STREAM_BUDGET_BYTES = 1 << 30


@xl.boundary
def compute_ensemble_mean(dataset, realization_name: str = REALIZATION,
                          skipna: bool = False):
  """Mean over `realization_name` of every variable that has it
  (scripts/compute_ensemble_mean.py:131: xbeam.Mean(REALIZATION_NAME, skipna)).

  float32 like xarray's mean of float32 data.  CUDA-tensor variables stay on
  the device (the result is a CUDA tensor K1 / K6 read in place); NumPy
  variables are uploaded, reduced and the (M times smaller) mean comes back.
  Variables without the dimension pass through.
  """
  ctx = _lib.default_context()
  out = xl.Dataset(attrs=dataset.attrs)
  for name in dataset.keys():
    v = dataset[name]
    if realization_name not in v.dims:
      out[name] = v
      continue
    dims = tuple(d for d in v.dims if d != realization_name)
    work = v.transpose(realization_name, *dims)
    data = work.data
    m = work.sizes[realization_name]
    shape = tuple(work.sizes[d] for d in dims)
    cells = int(np.prod(shape)) if shape else 1
    # one flat "field" per variable: the kernel walks it with a 64-bit
    # grid-stride loop, members `cells` elements apart
    slab = cells
    off = np.zeros(1, dtype=np.int64)
    coords = {k: c for k, c in work.coords.items()
              if realization_name not in c.dims}
    values, = _streamed.run_whole(
        [data], [(shape, np.float32)],
        lambda i, o: ctx.ens_mean(i[0], m, cells, off, slab, skipna, o[0]),
        dtype=np.float32)
    out[name] = xl.DataArray(values, dims, coords, name, v.attrs)
  return out


def _check_quantiles(quantiles) -> list:
  quantiles = [float(q) for q in quantiles]
  if any(not 0 <= q <= 1 for q in quantiles):  # NaN fails both comparisons
    raise ValueError(
        f'Expected all quantiles to be in [0, 1]. Found {quantiles=}')
  if not quantiles or len(quantiles) > _lib.MAX_QUANTILES:
    raise ValueError(f'between 1 and {_lib.MAX_QUANTILES} quantiles are '
                     f'supported per call (got {len(quantiles)})')
  return quantiles


def _variable_quantiles(v: xl.DataArray, reduce: list, quantiles: list,
                        skipna: bool):
  """The quantiles of `v` over the dims `reduce`: [nq, *preserved shape], a
  CUDA tensor for CUDA data, else NumPy.  Adjacent reduced dims are read in
  place as [outer][n][inner]; otherwise one transposed contiguous copy with
  the reduced dims in front is made first (torch on the device, NumPy on the
  host)."""
  if v.dtype not in (np.float32, np.float64):
    raise TypeError(f'variable {v.name!r} has dtype {v.dtype}: quantiles '
                    'take float32 or float64 data')
  pos = sorted(v.dims.index(d) for d in reduce)
  keep = [d for d in v.dims if d not in reduce]
  nsample = math.prod(v.sizes[d] for d in reduce)
  if nsample == 0:
    raise ValueError(f'variable {v.name!r}: cannot take quantiles over an '
                     f'empty reduction ({reduce})')
  perm = None
  if not pos:  # a 0-d variable: one sample
    nouter = ninner = 1
  elif pos[-1] - pos[0] == len(pos) - 1:
    nouter = math.prod(v.shape[:pos[0]])
    ninner = math.prod(v.shape[pos[-1] + 1:])
  else:
    nouter, ninner = 1, math.prod(v.sizes[d] for d in keep)
    perm = pos + [v.dims.index(d) for d in keep]
  out_shape = (len(quantiles),) + tuple(v.sizes[d] for d in keep)
  return _streamed.run('quantile', v.data,
                       (nouter, nsample, ninner, quantiles, skipna),
                       [(out_shape, np.float64)], QUANTILE_STREAM_BUDGET_BYTES,
                       perm=perm)[0]


@xl.boundary
def compute_quantiles_core(chunk, quantiles: Sequence[float], dim, *,
                           skipna: bool = False, name_suffix: str = ''):
  """`_evaluate_chunk_core` of scripts/compute_quantiles.py:168-183:
  `chunk.quantile(quantiles, dim=dim, skipna=skipna)` (method 'linear') with
  every variable `v` renamed `v + name_suffix`.

  Like xarray's Dataset.quantile: a float64 `quantile` dimension comes first,
  then the preserved dims in input order; coordinates along reduced dims are
  dropped; a variable with none of the reduced dims passes through; attrs
  are dropped.  The values are numpy's np.quantile / np.nanquantile bit for
  bit, as float64 (include/wb2b200.h, DESIGN.md section 8f).  CUDA-tensor
  variables give CUDA tensors; NumPy or memmap variables are streamed
  through the device in bands and give NumPy.  Reduced dims need not be
  adjacent: when they are not, the variable is copied once, transposed with
  the reduced dims in front (torch on the device, NumPy on the host)."""
  dims = [dim] if isinstance(dim, str) else list(dim)
  preserve_dims = set(d for d in chunk.dims if d not in dims)
  if not preserve_dims.issubset(set(chunk.dims)):
    raise ValueError(
        f'User specified dim={dims}, which results in preserved dims'
        f' {preserve_dims} , not being a subset of {set(chunk.dims)=}')
  quantiles = _check_quantiles(quantiles)
  missing = [d for d in dims if d not in chunk.dims]
  if missing:
    raise ValueError(f'Dimensions {tuple(missing)} not found in data '
                     f'dimensions {tuple(chunk.dims)}')
  coords = {k: c for k, c in chunk.coords.items()
            if not any(d in dims for d in c.dims)}
  coords[QUANTILE] = xl.Coord((QUANTILE,), np.asarray(quantiles, np.float64))
  out = xl.Dataset(coords=coords)
  for name in chunk.keys():
    v = chunk[name]
    reduce = [d for d in v.dims if d in dims]
    if not reduce and v.dims:
      out[name + name_suffix] = xl.DataArray(v.data, v.dims, attrs=v.attrs)
      continue
    values = _variable_quantiles(v, reduce, quantiles, skipna)
    out[name + name_suffix] = xl.DataArray(
        values, (QUANTILE,) + tuple(d for d in v.dims if d not in reduce))
  return out


@xl.boundary
def compute_quantiles(ds, quantiles: Sequence[float], dim, *,
                      skipna: bool = False, name_suffix: str = '',
                      variables: Optional[Sequence[str]] = None,
                      levels: Optional[Sequence] = None,
                      time_dim: str = 'time',
                      time_start: Optional[str] = '2020-01-01',
                      time_stop: Optional[str] = '2020-12-31'):
  """scripts/compute_quantiles.py `main` without Beam or zarr: the script's
  `_impose_data_selection` (variables, then [time_start, time_stop] on
  `time_dim` with both ends inclusive and the script's default range, then
  `levels` on `level`, each only where the dim exists), then
  `compute_quantiles_core`."""
  ds = _impose_data_selection(ds, variables, levels, time_dim, time_start,
                              time_stop)
  return compute_quantiles_core(ds, quantiles, dim, skipna=skipna,
                                name_suffix=name_suffix)


def _impose_data_selection(ds: xl.Dataset, variables, levels, time_dim,
                           time_start, time_stop) -> xl.Dataset:
  """`_impose_data_selection` of scripts/compute_quantiles.py and
  compute_averages.py: `variables`, then [time_start, time_stop] on
  `time_dim` with both ends inclusive, then `levels` on `level`, each only
  where the dim exists."""
  if variables is not None:
    ds = ds[list(variables)]
  if time_dim in ds.dims:
    index = pd.Index(ds.coords[time_dim].values)
    ds = ds.isel({time_dim: index.slice_indexer(time_start, time_stop)})
  if levels and 'level' in ds.dims:
    ds = ds.sel(level=[float(l) for l in levels])
  return ds


# -- means and raw moments over reduced dims (csrc/average.cu) -----------------
MOMENT = 'moment'
MOMENT_ORDERS = ('zeroth', 'first', 'second')
# device bytes of the two staging buffers of a host (NumPy) average call
AVERAGE_STREAM_BUDGET_BYTES = 1 << 30
_STATS = ('mean', 'mean_sq', 'frac')


def _average_layout(v: xl.DataArray, reduce: list):
  """The canonical (k0, r0, k1, r1, k2) of `v` reduced over `reduce`, the
  permutation that makes it one (None: `v` is read in place) and the reduced
  dims in sample order.  Adjacent dims of the same kind are merged; a reduced
  set of three or more runs is moved in front by one transposed copy."""
  runs = []  # [is_reduced, [dims]]
  for d in v.dims:
    r = d in reduce
    if runs and runs[-1][0] == r:
      runs[-1][1].append(d)
    else:
      runs.append([r, [d]])
  perm = None
  if sum(r for r, _ in runs) > 2:
    red = [d for d in v.dims if d in reduce]
    keep = [d for d in v.dims if d not in reduce]
    perm = [v.dims.index(d) for d in red + keep]
    runs = [[True, red]] + ([[False, keep]] if keep else [])
  # K R K or K R K R K; the last kept run is always k2, which the kernels
  # read coalesced across cells
  if runs[0][0]:
    runs.insert(0, [False, []])
  if runs[-1][0]:
    runs.append([False, []])
  if len(runs) == 3:
    runs[2:2] = [[False, []], [True, []]]
  shape = tuple(math.prod(v.sizes[d] for d in dims) for _, dims in runs)
  sample_dims = runs[1][1] + runs[3][1]
  return shape, perm, sample_dims


def _check_average(v: xl.DataArray, reduce):
  if not reduce:
    raise ValueError(f'variable {v.name!r}: the dims to average over are '
                     f'empty ({list(reduce)})')
  if v.dtype not in (np.float32, np.float64):
    raise TypeError(f'variable {v.name!r} has dtype {v.dtype}: averages '
                    'take float32 or float64 data')
  for d in reduce:
    if d not in v.dims:
      raise ValueError(f'variable {v.name!r} has no dimension {d!r} to '
                       f'average over (dims {v.dims})')
  if any(v.sizes[d] == 0 for d in reduce):
    raise ValueError(f'variable {v.name!r}: cannot average over an empty '
                     f'reduction ({reduce})')


def _variable_average(v: xl.DataArray, reduce: list, stats, *, skipna: bool,
                      weights=None, weight_dim: str = 'latitude'):
  """{stat: array} of `v` over the dims `reduce` for each stat of `stats`
  ('mean', 'mean_sq', 'frac'), shaped like the kept dims in input order: CUDA
  tensors for CUDA data, else NumPy (streamed through the device in bands).
  `weights` (a float64 vector along `weight_dim`, which must be reduced)
  multiplies every sample first; the divisor stays the sample count."""
  _check_average(v, reduce)
  shape, perm, sample_dims = _average_layout(v, reduce)
  wkw = {}
  if weights is not None:
    i = sample_dims.index(weight_dim)
    wkw = dict(weights=np.asarray(weights, np.float64),
               wdiv=math.prod(v.sizes[d] for d in sample_dims[i + 1:]))
  keep_shape = tuple(v.sizes[d] for d in v.dims if d not in reduce)
  dt = np.float64 if weights is not None else v.dtype
  dtypes = {'mean': dt, 'mean_sq': dt, 'frac': np.float64}
  res = _streamed.run(
      'average', v.data, (shape, skipna),
      [(keep_shape, dtypes[s]) if s in stats else None for s in _STATS],
      AVERAGE_STREAM_BUDGET_BYTES, perm=perm, **wkw)
  res = dict(zip(_STATS, res))
  return {s: res[s] for s in stats}


def _kept_coords(ds: xl.Dataset, dims) -> dict:
  return {k: c for k, c in ds.coords.items()
          if not any(d in dims for d in c.dims)}


@xl.boundary
def compute_averages(ds, averaging_dims: Sequence[str], *,
                     skipna: bool = False,
                     variables: Optional[Sequence[str]] = None,
                     levels: Optional[Sequence] = None,
                     time_dim: str = 'time',
                     time_start: Optional[str] = '2020-01-01',
                     time_stop: Optional[str] = '2020-12-31'):
  """scripts/compute_averages.py `main` without Beam or zarr: the script's
  `_impose_data_selection`, then per variable `v * weights` (when `latitude`
  is averaged: metrics.get_lat_weights of the selected dataset) followed by
  xbeam.Mean(averaging_dims, skipna).

  Like that Mean, the divisor is the number of samples counted (all of them,
  or the non-NaN ones with skipna), not the sum of the weights; with
  get_lat_weights (mean 1) and no NaN the two agree.  The result is float64
  when weighted (the reference's float32 * float64 product), else the data
  type; it keeps the other dims in input order, drops coordinates along
  averaged dims and has no attrs.  A variable without one of the averaging
  dims raises ValueError.  CUDA-tensor variables give CUDA tensors; NumPy or
  memmap variables are streamed through the device and give NumPy.  Sums are
  float64 in the order include/wb2b200.h fixes (DESIGN.md section 8g)."""
  ds = _impose_data_selection(ds, variables, levels, time_dim, time_start,
                              time_stop)
  dims = [averaging_dims] if isinstance(averaging_dims, str) else list(
      averaging_dims)
  weights = None
  if 'latitude' in dims:
    from weatherbench2_b200 import metrics  # pylint: disable=import-outside-toplevel
    weights = metrics.get_lat_weights(ds).values
  for name in ds.keys():
    _check_average(ds[name], dims)
  out = xl.Dataset(coords=_kept_coords(ds, dims))
  for name in ds.keys():
    v = ds[name]
    res = _variable_average(v, dims, ('mean',), skipna=skipna,
                            weights=weights)
    out[name] = xl.DataArray(res['mean'],
                             tuple(d for d in v.dims if d not in dims))
  return out


def _moment_stat(order: str) -> str:
  try:
    return _STATS[('first', 'second', 'zeroth').index(order)]
  except ValueError:
    raise NotImplementedError(f'Order {order} not implemented.') from None


@xl.boundary
def moment_reduce(obs, order: str = 'first',
                  reduce_dims: Sequence[str] = ('longitude', 'latitude'),
                  sel_kwargs: Optional[dict] = None):
  """`moment_reduce` of scripts/compute_statistical_moments.py: the mean over
  `reduce_dims` of the data (order 'first'), of its square rounded in the
  data type (np.square, 'second') or of its non-NaN mask ('zeroth': the
  fraction of non-NaN samples, float64).  Unweighted and NaN-skipping, as
  xarray's mean of float data is; other orders raise NotImplementedError."""
  stat = _moment_stat(order)
  if sel_kwargs:
    obs = obs.sel(sel_kwargs)
  dims = [reduce_dims] if isinstance(reduce_dims, str) else list(reduce_dims)
  for name in obs.keys():
    _check_average(obs[name], dims)
  out = xl.Dataset(coords=_kept_coords(obs, dims))
  for name in obs.keys():
    v = obs[name]
    res = _variable_average(v, dims, (stat,), skipna=True)
    out[name] = xl.DataArray(res[stat],
                             tuple(d for d in v.dims if d not in dims))
  return out


@xl.boundary
def compute_statistical_moments(obs, *, start_year: Optional[int] = 1990,
                                end_year: Optional[int] = 2020,
                                time_dim: str = 'time'):
  """scripts/compute_statistical_moments.py `main` without Beam or zarr: the
  years start_year..end_year (both inclusive) of `time_dim`, then per
  variable the zeroth, first and second raw moments over longitude and
  latitude (one read of the data for all three), then their mean over time.

  The spatial moments are kept in the dtypes the reference materialises (the
  data type, the data type, float64) before the time mean, which skips NaN
  steps.  The result has variables `{var}_{order}`, order-major as the
  script's template, with dims ('moment', *rest): `moment` has size 1 and no
  coordinate."""
  if start_year is not None and end_year is not None:
    index = pd.Index(obs.coords[time_dim].values)
    obs = obs.isel({time_dim: index.slice_indexer(str(start_year),
                                                  str(end_year))})
  space = ['longitude', 'latitude']
  gone = space + [time_dim]
  out = xl.Dataset(coords=_kept_coords(obs, gone))
  for name in obs.keys():
    _check_average(obs[name], gone)
  results = {}
  for name in obs.keys():
    v = obs[name]
    spatial = _variable_average(v, space, _STATS, skipna=True)
    sdims = tuple(d for d in v.dims if d not in space)
    rest = tuple(d for d in sdims if d != time_dim)
    for order in MOMENT_ORDERS:
      s = xl.DataArray(spatial[_moment_stat(order)], sdims, name=name)
      m = _variable_average(s, [time_dim], ('mean',), skipna=True)['mean']
      results[(order, name)] = (m.reshape((1,) + tuple(m.shape)), rest)
  for order in MOMENT_ORDERS:
    for name in obs.keys():
      values, rest = results[(order, name)]
      out[f'{name}_{order}'] = xl.DataArray(values, (MOMENT,) + rest)
  return out

"""Reindexing in time without a GPU: weatherbench2_b200.reindexing end to end
on `fake_ctx_reindex` (NumPy interpreting the C-ABI arguments) against the
label-by-label oracle (tests/reindex_oracle.py) and the reference's own
results (tests/golden/reference_reindex_vectors.npz, made by
tests/golden/make_reindex_vectors.py): the sampler bit for bit in every
branch, the forecast offset and spacing, the expected arrays of the
reference's index_on_valid_time and expand_climatology tests, every dim
order, the renames, the properties of the reference's standard workflow
test, and every error.  tests/test_reindex_gpu.py runs the operations through
the CUDA kernels."""
import importlib
import itertools
import json
import os
import sys

import numpy as np
import pandas as pd
import pytest

import fake_ctx_reindex
import reindex_oracle as ro

HERE = os.path.dirname(os.path.abspath(__file__))
VECTORS = os.path.join(HERE, 'golden', 'reference_reindex_vectors.npz')
FAKE_XARRAY = os.path.join(HERE, 'fake_xarray')


def _vectors():
  with np.load(VECTORS) as z:
    return {k: z[k] for k in z.files}


V = _vectors()


def _names(kind):
  return sorted({k.split('|')[1] for k in V if k.startswith(kind + '|')})


def fake_run(fn, *args, **kw):
  with fake_ctx_reindex.installed() as fake:
    return fn(*args, **kw), fake


def _xl():
  from weatherbench2_b200 import xarray_lite as xl
  return xl


# -- the sampler and the plan functions against the reference -------------------
@pytest.mark.parametrize('name', _names('sampler'))
def test_sampled_init_times_match_the_reference_bit_for_bit(name):
  from weatherbench2_b200 import reindexing as ri
  kw = json.loads(str(V[f'sampler|{name}|args']))
  times = pd.DatetimeIndex(kw.pop('times'))
  err = V.get(f'sampler|{name}|error')
  if err is not None:
    kind, msg = str(err).split('|', 1)
    with pytest.raises(ValueError) as info:
      ri.get_sampled_init_times(times, **kw)
    if kind == 'ValueError':
      assert str(info.value) == msg
    return
  got = ri.get_sampled_init_times(times, **kw)
  assert got.dtype == np.dtype('datetime64[ns]')
  np.testing.assert_array_equal(got.view(np.int64), V[f'sampler|{name}|result'])


def test_the_vectors_cover_every_sampler_branch():
  cases = [json.loads(str(V[f'sampler|{n}|args'])) for n in _names('sampler')
           if f'sampler|{n}|result' in V]
  assert len(_names('sampler')) >= 40
  for edge in ('WRAP_YEAR', 'REFLECT_RANGE', 'NO_EDGE'):
    for repl in (True, False):
      assert any(c['initial_time_edge_behavior'] == edge and
                 c['with_replacement'] == repl for c in cases)
  assert any(c['ensemble_size'] == -1 for c in cases)
  assert any(c['sample_hold_days'] for c in cases)
  for repl in (True, False):
    assert any(c['leave_out_if_in_climatology'] and c['with_replacement'] == repl
               and c['num_years_to_exclude'] for c in cases)


@pytest.mark.parametrize('name', _names('ensemble_size'))
def test_ensemble_size_matches_the_reference(name):
  from weatherbench2_b200 import reindexing as ri
  args = json.loads(str(V[f'ensemble_size|{name}|args']))
  if f'ensemble_size|{name}|error' in V:
    with pytest.raises(ValueError):  # the reference: flags.ValidationError
      ri.get_ensemble_size(*args)
    return
  assert ri.get_ensemble_size(*args) == int(V[f'ensemble_size|{name}|result'])


@pytest.mark.parametrize('name', _names('spacing'))
def test_forecast_offset_and_spacing_match_the_reference(name):
  from weatherbench2_b200 import reindexing as ri
  init = V[f'spacing|{name}|init'].view('datetime64[ns]')
  lead = V[f'spacing|{name}|lead'].view('timedelta64[ns]')
  if f'spacing|{name}|error' in V:
    with pytest.raises(ValueError):
      ri.get_forecast_offset_and_spacing(init, lead)
    return
  assert ri.get_forecast_offset_and_spacing(init, lead) == tuple(
      V[f'spacing|{name}|result'])


# -- index_on_valid_time --------------------------------------------------------
IVT_CASES = {'no_offset_delta': 'valid_and_delta',
             'no_offset_init': 'valid_and_init',
             'offset_delta': 'valid_and_delta', 'offset_init': 'valid_and_init'}


def _ivt_input(x, lead_hours, dims=('time', 'prediction_timedelta')):
  xl = _xl()
  init = pd.date_range('2000-01-01T00', periods=x.shape[0], freq='12h').values
  leads = np.asarray(lead_hours, 'timedelta64[h]').astype('timedelta64[ns]')
  return xl.Dataset({'foo': (dims, x)},
                    {'time': init, 'prediction_timedelta': leads})


@pytest.mark.parametrize('case', sorted(IVT_CASES))
def test_index_on_valid_time_gives_the_reference_tests_arrays(case):
  from weatherbench2_b200 import reindexing as ri
  ds = _ivt_input(V[f'ivt|{case}|x'], V[f'ivt|{case}|lead_hours'])
  mode = IVT_CASES[case]
  out, _ = fake_run(ri.index_on_valid_time, ds, desired_time_dims=mode)
  foo = out['foo']
  assert foo.dtype == np.float32
  base = np.datetime64('2000-01-01T00', 'ns')
  want_time = base + V[f'ivt|{case}|want_time_hours'].astype('timedelta64[h]')
  np.testing.assert_array_equal(out.coords['time'].values, want_time)
  other = V[f'ivt|{case}|want_other_hours'].astype('timedelta64[h]')
  if mode == 'valid_and_delta':
    assert foo.dims == ('time', 'prediction_timedelta')
    np.testing.assert_array_equal(out.coords['prediction_timedelta'].values,
                                  other)
  else:
    assert foo.dims == ('init', 'time')
    np.testing.assert_array_equal(out.coords['init'].values, base + other)
  np.testing.assert_array_equal(foo.values,
                                V[f'ivt|{case}|want'].astype(np.float32))


IVT_DIMS = [('time', 'prediction_timedelta', 'level', 'cell'),
            ('prediction_timedelta', 'time', 'level', 'cell'),
            ('level', 'time', 'cell', 'prediction_timedelta'),
            ('cell', 'prediction_timedelta', 'level', 'time')]


def ivt_case(dims, mode, dtype, seed, lead_hours=(0, 6, 12, 18, 24, 30, 36),
             ncell=5, ninit=4, to_device=None):
  """Runs one index_on_valid_time case and checks it against the oracle;
  returns the result."""
  from weatherbench2_b200 import reindexing as ri
  xl = _xl()
  sizes = {'time': ninit, 'prediction_timedelta': len(lead_hours), 'level': 3,
           'cell': ncell}
  rs = np.random.RandomState(seed)
  x = rs.normal(size=[sizes[d] for d in dims])
  x = (x * 1000).astype(dtype) if np.dtype(dtype).kind == 'i' else x.astype(
      dtype)
  init = pd.date_range('2000-01-01', periods=ninit, freq='12h').values
  leads = np.asarray(lead_hours, 'timedelta64[h]').astype('timedelta64[ns]')
  ds = xl.Dataset({'v': (dims, x), 'w': (dims, x[::-1].copy())},
                  {'time': init, 'prediction_timedelta': leads,
                   'level': np.array([500, 700, 850])})
  if to_device is not None:
    ds = to_device(ds)
  out = ri.index_on_valid_time(ds, desired_time_dims=mode)
  off, sp = ri.get_forecast_offset_and_spacing(init, leads)
  for name, src in (('v', x), ('w', x[::-1])):
    want, wdims, times = ro.index_on_valid_time(src, dims, init, leads, off, sp,
                                                mode)
    assert out[name].dims == wdims
    np.testing.assert_array_equal(out.coords['time'].values, times)
    np.testing.assert_array_equal(np.asarray(out[name].values), want)
    assert out[name].dtype == np.float32
  np.testing.assert_array_equal(out.coords['level'].values, [500, 700, 850])
  return out


@pytest.mark.parametrize('dims,mode', list(itertools.product(
    IVT_DIMS, ['valid_and_delta', 'valid_and_init'])))
@pytest.mark.parametrize('dtype', [np.float32, np.float64, np.int64])
def test_index_on_valid_time_every_dim_order_matches_the_oracle(dims, mode,
                                                                 dtype):
  fake_run(ivt_case, dims, mode, dtype, 1)


def test_index_on_valid_time_lead_offset_and_daily_inits():
  for mode in ('valid_and_delta', 'valid_and_init'):
    fake_run(ivt_case, IVT_DIMS[0], mode, np.float32, 2,
             lead_hours=tuple(range(6, 49, 6)))


def test_index_on_valid_time_errors():
  from weatherbench2_b200 import reindexing as ri
  xl = _xl()
  x = np.zeros((3, 4, 2), np.float32)
  coords = {'time': pd.date_range('2000-01-01', periods=3, freq='12h').values,
            'prediction_timedelta': np.arange(4) * np.timedelta64(6, 'h')}
  ds = xl.Dataset({'a': (('time', 'prediction_timedelta', 'c'), x),
                   'b': (('prediction_timedelta', 'time', 'c'),
                         x.transpose(1, 0, 2).copy())}, coords)
  with pytest.raises(ValueError, match='different axes'):
    fake_run(ri.index_on_valid_time, ds)
  ds = xl.Dataset({'a': (('time', 'prediction_timedelta', 'c'), x),
                   'static': (('c',), np.zeros(2, np.float32))}, coords)
  with pytest.raises(ValueError, match="'static'"):
    fake_run(ri.index_on_valid_time, ds)
  with pytest.raises(ValueError, match='Unhandled'):
    fake_run(ri.index_on_valid_time, ds, desired_time_dims='valid')
  one = xl.Dataset({'a': (('time', 'prediction_timedelta'), x[:1, :, 0])},
                   {'time': coords['time'][:1],
                    'prediction_timedelta': coords['prediction_timedelta']})
  with pytest.raises(ValueError):
    fake_run(ri.index_on_valid_time, one)
  ds = xl.Dataset({'a': (('time', 'prediction_timedelta', 'c'),
                         x.astype(np.float16))}, coords)
  with pytest.raises(TypeError, match="'a'"):
    fake_run(ri.index_on_valid_time, ds)


# -- expand_climatology -----------------------------------------------------------
def _climatology(dims, hours=(0, 6, 12, 18), ndoy=366, seed=0, dtype=np.float32,
                 to_device=None):
  xl = _xl()
  sizes = {'hour': len(hours), 'dayofyear': ndoy, 'level': 2, 'latitude': 3,
           'longitude': 4}
  rs = np.random.RandomState(seed)
  x = rs.normal(size=[sizes[d] for d in dims]).astype(dtype)
  coords = {'dayofyear': np.arange(1, ndoy + 1), 'level': np.array([500, 850]),
            'latitude': np.linspace(-60, 60, 3),
            'longitude': np.arange(4) * 90.0}
  if 'hour' in dims:
    coords['hour'] = np.asarray(hours)
  ds = xl.Dataset({'z': (dims, x), 't2m': (dims, x * 2)}, coords)
  return (to_device(ds) if to_device else ds), x


CLIM_DIMS = [('hour', 'dayofyear', 'level', 'latitude', 'longitude'),
             ('dayofyear', 'hour', 'level', 'latitude', 'longitude'),
             ('level', 'dayofyear', 'hour', 'longitude', 'latitude'),
             ('latitude', 'hour', 'longitude', 'dayofyear', 'level'),
             ('dayofyear', 'level', 'latitude', 'longitude')]


def expand_case(dims, start, stop, dtype=np.float32, to_device=None):
  from weatherbench2_b200 import reindexing as ri
  ds, x = _climatology(dims, dtype=dtype, to_device=to_device)
  out = ri.expand_climatology(ds, time_start=start, time_stop=stop)
  step = '6h' if 'hour' in dims else '1D'
  times = pd.date_range(start, stop, freq=step)
  np.testing.assert_array_equal(out.coords['time'].values, times.values)
  for name, src in (('z', x), ('t2m', x * 2)):
    want, wdims = ro.expand_climatology(src, dims, np.arange(1, 367),
                                        np.array([0, 6, 12, 18]), times)
    assert out[name].dims == wdims
    np.testing.assert_array_equal(np.asarray(out[name].values), want)
    assert out[name].dtype == dtype
  assert 'dayofyear' not in out.coords and 'hour' not in out.coords
  return out


@pytest.mark.parametrize('dims', CLIM_DIMS, ids=lambda d: '-'.join(d))
@pytest.mark.parametrize('dtype', [np.float32, np.float64])
def test_expand_climatology_every_dim_order_matches_the_oracle(dims, dtype):
  fake_run(expand_case, dims, '2019-12-01', '2020-03-30', dtype)


def test_expand_climatology_gives_the_reference_tests_arrays():
  from weatherbench2_b200 import reindexing as ri
  xl = _xl()
  clim = V['expand|clim']
  dims = ('hour', 'dayofyear', 'level', 'latitude', 'longitude')
  ds = xl.Dataset({'geopotential': (dims, clim)},
                  {'hour': np.arange(0, 24, 6), 'dayofyear': np.arange(1, 367),
                   'level': np.array([500, 850]), 'latitude': np.arange(3.0),
                   'longitude': np.arange(2.0)})
  out, fake = fake_run(ri.expand_climatology, ds, time_start='2019-12-01',
                       time_stop='2020-03-30')
  np.testing.assert_array_equal(out.coords['time'].values.view(np.int64),
                                V['expand|time_ns'])
  np.testing.assert_array_equal(out['geopotential'].values, V['expand|want'])
  # one gather per variable, of one (level, lat, lon) slab per time
  assert fake.calls == [('slab_gather_host', V['expand|want'].shape[0], 12,
                         4 << 30)]


def test_expand_climatology_errors():
  from weatherbench2_b200 import reindexing as ri
  ds365, _ = _climatology(CLIM_DIMS[0], ndoy=365)
  with pytest.raises(KeyError):  # 2020-12-31 is day 366
    fake_run(ri.expand_climatology, ds365, time_start='2020-12-30',
             time_stop='2020-12-31')
  ds, _ = _climatology(CLIM_DIMS[0], hours=(0, 12))
  with pytest.raises(KeyError):  # hour 6 is off the 12-hourly grid
    fake_run(ri.expand_climatology, ds, time_start='2020-01-01T06',
             time_stop='2020-01-02')
  one, _ = _climatology(CLIM_DIMS[0], hours=(0,))
  with pytest.raises(ValueError, match='two hours'):
    fake_run(ri.expand_climatology, one, time_start='2020-01-01',
             time_stop='2020-01-02')
  xl = _xl()
  ds, _ = _climatology(CLIM_DIMS[0])
  ds['lsm'] = xl.DataArray(np.zeros((3, 4), np.float32),
                           ('latitude', 'longitude'))
  with pytest.raises(ValueError, match="'lsm'"):
    fake_run(ri.expand_climatology, ds, time_start='2020-01-01',
             time_stop='2020-01-02')
  out, _ = fake_run(ri.expand_climatology, ds, time_start='2020-01-01',
                    time_stop='2020-01-02', variables=['z'])
  assert list(out.keys()) == ['z']


# -- probabilistic climatological forecasts -----------------------------------------
def _truth(dims=('time', 'level', 'latitude', 'longitude'), start='1990-01-01',
           stop='1993-12-31', freq='6h', seed=0, dtype=np.float32,
           growing=False, to_device=None, time_dim='time'):
  xl = _xl()
  times = pd.date_range(start, stop, freq=freq)
  sizes = {time_dim: times.size, 'level': 2, 'latitude': 3, 'longitude': 2}
  shape = [sizes[d] for d in dims]
  if growing:  # value = time step index, in every cell
    x = np.broadcast_to(np.arange(times.size).reshape(
        [-1 if d == time_dim else 1 for d in dims]), shape).astype(dtype)
  else:
    x = np.random.RandomState(seed).normal(size=shape).astype(dtype)
  ds = xl.Dataset({'t': (dims, np.ascontiguousarray(x))},
                  {time_dim: times.values, 'level': np.array([500, 850]),
                   'latitude': np.arange(3.0), 'longitude': np.arange(2.0)})
  return (to_device(ds) if to_device else ds), x, times


PROB_KW = dict(initial_time_start='1991-01-01', initial_time_end='1991-01-05',
               climatology_start_year=1991, climatology_end_year=1992,
               forecast_duration='2 days', ensemble_size=3, day_window_size=5,
               add_source_time=True, seed=3)

TRUTH_DIMS = [('time', 'level', 'latitude', 'longitude'),
              ('level', 'time', 'latitude', 'longitude'),
              ('latitude', 'longitude', 'level', 'time'),
              ('longitude', 'time', 'latitude', 'level')]


def prob_case(dims, to_device=None, dtype=np.float32, **kw):
  from weatherbench2_b200 import reindexing as ri
  kw = dict(PROB_KW, **kw)
  time_dim = kw.get('time_dim', 'time')
  dims = tuple(time_dim if d == 'time' else d for d in dims)
  ds, x, times = _truth(dims, dtype=dtype, to_device=to_device,
                        time_dim=time_dim)
  out = ri.compute_probabilistic_climatological_forecasts(ds, **kw)
  sample_kw = {k: kw[k] for k in (
      'climatology_start_year', 'climatology_end_year', 'day_window_size',
      'ensemble_size', 'seed')}
  inits = pd.date_range(kw['initial_time_start'], kw['initial_time_end'],
                        freq=kw.get('initial_time_spacing', '6h'))
  sampled = ri.get_sampled_init_times(inits, **sample_kw)
  deltas = pd.timedelta_range('0 days', kw['forecast_duration'],
                              freq=kw.get('timedelta_spacing', '6h'))
  want, wdims = ro.sample_forecasts(x, dims, times.values, sampled, deltas,
                                    time_dim)
  real = kw.get('realization_name', 'realization')
  wdims = (real,) + wdims[1:]
  assert out['t'].dims == wdims
  assert out['t'].dtype == dtype
  np.testing.assert_array_equal(np.asarray(out['t'].values), want)
  st = out['source_time']
  assert st.dims == wdims[:3] and st.dtype == np.dtype('datetime64[ns]')
  np.testing.assert_array_equal(
      st.values, sampled[:, None, :] + deltas.values[None, :, None])
  np.testing.assert_array_equal(out.coords[real].values, np.arange(3))
  np.testing.assert_array_equal(out.coords[time_dim].values, inits.values)
  np.testing.assert_array_equal(out.coords['prediction_timedelta'].values,
                                deltas.values)
  return out


@pytest.mark.parametrize('dims', TRUTH_DIMS, ids=lambda d: '-'.join(d))
@pytest.mark.parametrize('dtype', [np.float32, np.float64])
def test_probabilistic_forecasts_every_dim_order_match_the_oracle(dims, dtype):
  fake_run(prob_case, dims, dtype=dtype)


def test_probabilistic_forecasts_time_dim_and_realization_renames():
  fake_run(prob_case, TRUTH_DIMS[1], time_dim='valid', realization_name='number')


def test_probabilistic_forecasts_standard_workflow_properties():
  """The reference's test_standard_workflow: on a dataset that grows by one
  each step, member m's forecast from init j at lead d is d steps past its
  start, and source_time is the time read."""
  from weatherbench2_b200 import reindexing as ri
  ds, _, times = _truth(growing=True, dtype=np.float64)
  out, _ = fake_run(ri.compute_probabilistic_climatological_forecasts, ds,
                    **dict(PROB_KW, ensemble_size=4, sample_hold_days=2,
                           initial_time_edge_behavior='REFLECT_RANGE',
                           initial_time_end='1991-01-20'))
  v = out['t'].values  # (realization, delta, time, level, lat, lon)
  nd = v.shape[1]
  np.testing.assert_array_equal(v - v[:, :1], np.broadcast_to(
      np.arange(nd).reshape(1, -1, 1, 1, 1, 1), v.shape))
  st = out['source_time'].values
  np.testing.assert_array_equal(times.values[v[..., 0, 0, 0].astype(int)], st)
  np.testing.assert_array_equal(st - st[:, :1], np.broadcast_to(
      (np.arange(nd) * np.timedelta64(6, 'h')).astype('timedelta64[ns]')
      .reshape(1, -1, 1), st.shape))


def test_sample_forecasts_core_takes_any_columns_of_one_table():
  from weatherbench2_b200 import reindexing as ri
  ds, _, _ = _truth()
  inits = pd.date_range('1991-03-01', '1991-03-10', freq='12h')
  sampled = ri.get_sampled_init_times(
      inits, climatology_start_year=1991, climatology_end_year=1992,
      ensemble_size=3, seed=5)
  deltas = pd.timedelta_range('0 days', '1 days', freq='6h')
  whole, _ = fake_run(ri.sample_forecasts_core, ds, sampled, inits, deltas)
  for cols in (slice(0, 7), slice(7, None), [3, 11, 1]):
    part, _ = fake_run(ri.sample_forecasts_core, ds, sampled[:, cols],
                       inits[cols], deltas)
    np.testing.assert_array_equal(part['t'].values,
                                  whole['t'].values[:, :, cols])


def test_probabilistic_forecasts_select_variables_and_levels():
  from weatherbench2_b200 import reindexing as ri
  ds, x, _ = _truth()
  ds['u'] = ds['t'] * 2
  out, _ = fake_run(ri.compute_probabilistic_climatological_forecasts, ds,
                    **dict(PROB_KW, variables=['u'], levels=['850'],
                           add_source_time=False))
  assert list(out.keys()) == ['u']
  np.testing.assert_array_equal(out.coords['level'].values, [850])
  assert out['u'].shape == (3, 9, 17, 1, 3, 2)


def test_probabilistic_forecasts_errors():
  from weatherbench2_b200 import reindexing as ri
  ds, _, _ = _truth()
  prob = ri.compute_probabilistic_climatological_forecasts
  with pytest.raises(ValueError, match='missing_times'):
    fake_run(prob, ds, **dict(PROB_KW, climatology_end_year=1994))
  with pytest.raises(ValueError, match='1 year before/after'):
    fake_run(prob, ds, **dict(PROB_KW, climatology_end_year=1994,
                              sample_hold_days=1))
  for kw, match in ((dict(timedelta_spacing='5h'), 'neither|multiple of'),
                    (dict(timedelta_spacing='3h'), 'not a multiple of input'),
                    (dict(initial_time_spacing='30h',
                          timedelta_spacing='30h'), 'multiple or divisor'),
                    (dict(ensemble_size=0), 'positive integer'),
                    (dict(ensemble_size=-1, leave_out_if_in_climatology=True),
                     'not supported')):
    with pytest.raises(ValueError, match=match):
      fake_run(prob, ds, **dict(PROB_KW, **kw))
  xl = _xl()
  lead = xl.Dataset({'t': (('time', 'prediction_timedelta'),
                           np.zeros((4, 2), np.float32))},
                    {'time': pd.date_range('1991-01-01', periods=4,
                                           freq='6h').values,
                     'prediction_timedelta': np.arange(2) * np.timedelta64(
                         6, 'h')})
  with pytest.raises(ValueError, match='already had prediction_timedelta'):
    fake_run(prob, lead, **dict(PROB_KW, initial_time_end='1991-01-01'))
  ds['lsm'] = xl.DataArray(np.zeros((3, 2), np.float32),
                           ('latitude', 'longitude'))
  with pytest.raises(ValueError, match="'lsm'"):
    fake_run(prob, ds, **PROB_KW)
  uneven = ds.isel(time=np.r_[0:10, 11:4000])
  with pytest.raises(ValueError, match='Non-unique spacing'):
    fake_run(prob, uneven, **PROB_KW)


# -- the entries' contract, and native xarray ------------------------------------
def test_fake_entry_refuses_an_invalid_table():
  from weatherbench2_b200 import _lib
  src = np.arange(10, dtype=np.float32)
  with pytest.raises(_lib.Wb2Error):
    fake_ctx_reindex.gather(src, 4, [0, 7], np.float32)
  got = fake_ctx_reindex.gather(src, 4, [6, -1], np.float64)
  np.testing.assert_array_equal(got[0], [6, 7, 8, 9])
  assert np.isnan(got[1]).all()


@pytest.fixture
def xr(monkeypatch):
  monkeypatch.syspath_prepend(FAKE_XARRAY)
  sys.modules.pop('xarray', None)
  mod = importlib.import_module('xarray')
  yield mod
  sys.modules.pop('xarray', None)


def test_native_xarray_in_gives_native_xarray_out(xr):
  from weatherbench2_b200 import reindexing as ri
  from weatherbench2_b200 import xarray_lite as xl
  lite = _ivt_input(V['ivt|no_offset_delta|x'].astype(np.float32),
                    V['ivt|no_offset_delta|lead_hours'])
  ds = xl.to_xarray(lite)
  assert isinstance(ds, xr.Dataset)
  out, _ = fake_run(ri.index_on_valid_time, ds)
  assert isinstance(out, xr.Dataset)
  np.testing.assert_array_equal(
      out['foo'].values, V['ivt|no_offset_delta|want'].astype(np.float32))
  clim, _ = _climatology(CLIM_DIMS[0])
  out, _ = fake_run(ri.expand_climatology, xl.to_xarray(clim),
                    time_start='2020-01-01', time_stop='2020-01-03')
  assert isinstance(out, xr.Dataset)
  truth, _, _ = _truth()
  out, _ = fake_run(ri.compute_probabilistic_climatological_forecasts,
                    xl.to_xarray(truth), **PROB_KW)
  assert isinstance(out, xr.Dataset)

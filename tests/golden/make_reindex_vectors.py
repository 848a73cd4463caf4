#!/usr/bin/env python
"""Runs the REFERENCE's own time samplers and plan functions
(<reference>/scripts/compute_probabilistic_climatological_forecasts.py:
`_get_sampled_init_times`, `_get_ensemble_size`;
<reference>/scripts/index_on_valid_time.py: `get_forecast_offset_and_spacing`
-- imported, not copied) on the argument sets below and stores their results,
or the type and message of the error they raise, in
reference_reindex_vectors.npz.  It also stores, as data, the expected arrays
of the reference's index_on_valid_time_test.py (its four cases) and a seeded
expand_climatology_test.py case (a 6-hourly climatology over 2019-12-01 to
2020-03-30, the expected values looked up by label as the test's `sel` does).

The scripts define absl flags at import, and absl refuses a flag defined
twice, so each script runs in a subprocess of its own, on
tests/golden/xarray_shim (the scripts import xarray, apache_beam and
xarray_beam at module level; the functions used here never call them).
tests/test_reindex_cpu.py holds weatherbench2_b200.reindexing to these
vectors bit for bit; only this script reads the reference.

Run:  python tests/golden/make_reindex_vectors.py <reference checkout>
"""
import json
import os
import subprocess
import sys

import numpy as np
import pandas as pd

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, 'reference_reindex_vectors.npz')


def sampler_cases():
  """name -> keyword arguments of _get_sampled_init_times (output_times as
  (start, end, freq) of pd.date_range)."""
  base = dict(times=('2020-01-01', '2020-01-10', '12h'),
              climatology_start_year=1990, climatology_end_year=1999,
              day_window_size=15, ensemble_size=4, with_replacement=True,
              sample_hold_days=0, initial_time_edge_behavior='WRAP_YEAR',
              leave_out_if_in_climatology=False, num_years_to_exclude=0,
              seed=802701)
  leap_dec = ('2019-12-20', '2020-01-12', '6h')
  feb = ('2020-02-20', '2020-03-05', '1D')
  odd_min = ('2020-06-01T03:30', '2020-06-03T03:30', '6h')
  cases = {}
  for edge in ('WRAP_YEAR', 'REFLECT_RANGE', 'NO_EDGE'):
    for repl in (True, False):
      for times, tag in ((base['times'], 'jan'), (leap_dec, 'dec'),
                         (feb, 'feb')):
        cases[f'{edge}_{"repl" if repl else "norepl"}_{tag}'] = dict(
            base, times=times, initial_time_edge_behavior=edge,
            with_replacement=repl, seed=len(cases) + 7)
  cases.update({
      'all_combinations': dict(base, ensemble_size=-1, day_window_size=4,
                               climatology_end_year=1992),
      'all_combinations_norepl': dict(base, ensemble_size=-1,
                                      day_window_size=3,
                                      climatology_end_year=1993,
                                      with_replacement=False),
      'even_window': dict(base, day_window_size=10),
      'window_1': dict(base, day_window_size=1),
      'window_728': dict(base, day_window_size=728, ensemble_size=3),
      'one_year_reflect': dict(base, climatology_start_year=2000,
                               climatology_end_year=2000,
                               initial_time_edge_behavior='REFLECT_RANGE',
                               times=leap_dec),
      'minutes_dropped': dict(base, times=odd_min),
      'hold_2d': dict(base, sample_hold_days=2, times=('2020-01-01',
                                                       '2020-01-20', '12h')),
      'hold_5d_reflect': dict(base, sample_hold_days=5,
                              initial_time_edge_behavior='REFLECT_RANGE',
                              times=('2020-12-01', '2021-01-10', '1D')),
      'hold_minutes': dict(base, sample_hold_days=1, times=odd_min),
      'leave_out_repl': dict(base, leave_out_if_in_climatology=True,
                             climatology_end_year=2022,
                             times=('2019-12-28', '2020-01-04', '1D'),
                             num_years_to_exclude=1),
      'leave_out_norepl': dict(base, leave_out_if_in_climatology=True,
                               with_replacement=False,
                               climatology_end_year=2022,
                               times=('1995-12-28', '1996-01-03', '1D'),
                               num_years_to_exclude=2),
      'leave_out_outside': dict(base, leave_out_if_in_climatology=True,
                                num_years_to_exclude=3),
      'single_time': dict(base, times=('2020-03-01', '2020-03-01', '1D')),
      'many_members': dict(base, ensemble_size=40, times=leap_dec),
      # errors
      'err_window_0': dict(base, day_window_size=0),
      'err_window_729': dict(base, day_window_size=729),
      'err_ensemble_0': dict(base, ensemble_size=0),
      'err_ensemble_minus1_leave_out': dict(base, ensemble_size=-1,
                                            leave_out_if_in_climatology=True),
      'err_empty_pool': dict(base, climatology_start_year=2000,
                             climatology_end_year=1999),
      'err_no_years_left': dict(base, leave_out_if_in_climatology=True,
                                climatology_start_year=2020,
                                climatology_end_year=2020),
      'err_not_enough_years': dict(base, leave_out_if_in_climatology=True,
                                   with_replacement=False, ensemble_size=40,
                                   climatology_end_year=2022),
      'err_norepl_too_many': dict(base, with_replacement=False,
                                  ensemble_size=200, day_window_size=5,
                                  climatology_end_year=1992),
      'err_edge': dict(base, initial_time_edge_behavior='CLAMP'),
      'err_hold_not_multiple': dict(base, sample_hold_days=1,
                                    times=('2020-01-01', '2020-01-05', '5h')),
      'err_hold_uneven': dict(base, sample_hold_days=2, times=[
          '2020-01-01', '2020-01-02', '2020-01-04']),
  })
  return cases


def ensemble_size_cases():
  return {'explicit': (5, 1990, 2000, 15, False),
          'all': (-1, 1990, 1999, 15, False),
          'all_even': (-1, 2001, 2003, 4, False),
          'err_zero': (0, 1990, 2000, 15, False),
          'err_negative': (-2, 1990, 2000, 15, False),
          'err_all_leave_out': (-1, 1990, 2000, 15, True)}


def spacing_cases():
  """name -> (init times (start, periods, freq), leads (hours))."""
  return {'no_offset': (('2000-01-01', 4, '12h'), [0, 6, 12, 18, 24]),
          'offset': (('2000-01-01', 4, '12h'), [6, 12, 18, 24]),
          'daily_6h': (('2000-01-01', 5, '1D'), list(range(0, 241, 6))),
          'same_step': (('2000-01-01', 3, '6h'), [0, 6, 12]),
          'hourly_offset': (('2000-01-01', 3, '3h'), [1, 2, 3, 4, 5]),
          'err_uneven_init': ([0, 12, 36], [0, 6, 12]),
          'err_uneven_lead': (('2000-01-01', 3, '12h'), [0, 6, 18]),
          'err_not_multiple': (('2000-01-01', 3, '12h'), [0, 5, 10]),
          'err_single_init': (('2000-01-01', 1, '12h'), [0, 6, 12]),
          'err_offset_missing': (('2000-01-01', 3, '12h'), [18, 24, 30])}


def _times(spec):
  if isinstance(spec, tuple):
    return pd.date_range(*spec[:2], freq=spec[2]).as_unit('ns')
  return pd.DatetimeIndex(spec).as_unit('ns')


def _init_times(spec):
  if isinstance(spec, tuple):
    return pd.date_range(spec[0], periods=spec[1],
                         freq=spec[2]).values.astype('datetime64[ns]')
  return (np.datetime64('2000-01-01', 'ns') +
          np.asarray(spec, 'timedelta64[h]')).astype('datetime64[ns]')


def _error(e):
  return f'{type(e).__name__}|{e}'


def run_probabilistic(reference):
  sys.argv = sys.argv[:1]
  from scripts import compute_probabilistic_climatological_forecasts as m
  out = {}
  for name, kw in sampler_cases().items():
    kw = dict(kw)
    times = _times(kw.pop('times'))
    out[f'sampler|{name}|args'] = np.array(json.dumps(
        dict(kw, times=[str(t) for t in times])))
    try:
      res = m._get_sampled_init_times(output_times=times, **kw)
      out[f'sampler|{name}|result'] = np.asarray(res, 'datetime64[ns]').view(
          np.int64)
    except Exception as e:  # pylint: disable=broad-except
      out[f'sampler|{name}|error'] = np.array(_error(e))
  for name, args in ensemble_size_cases().items():
    out[f'ensemble_size|{name}|args'] = np.array(json.dumps(args))
    try:
      out[f'ensemble_size|{name}|result'] = np.array(m._get_ensemble_size(*args))
    except Exception as e:  # pylint: disable=broad-except
      out[f'ensemble_size|{name}|error'] = np.array(_error(e))
  return out


def run_valid_time(reference):
  sys.argv = sys.argv[:1]
  from scripts import index_on_valid_time as m
  out = {}
  for name, (init, leads) in spacing_cases().items():
    it = _init_times(init)
    lt = np.asarray(leads, 'timedelta64[h]').astype('timedelta64[ns]')
    out[f'spacing|{name}|init'] = it.view(np.int64)
    out[f'spacing|{name}|lead'] = lt.view(np.int64)
    try:
      out[f'spacing|{name}|result'] = np.array(
          m.get_forecast_offset_and_spacing(it, lt))
    except Exception as e:  # pylint: disable=broad-except
      out[f'spacing|{name}|error'] = np.array(_error(e))
  return out


def reference_test_arrays():
  """The expected arrays of index_on_valid_time_test.py and a seeded
  expand_climatology_test.py case."""
  nan = np.nan
  src = np.arange(1, 21).reshape(4, 5)
  out = {
      'ivt|no_offset_delta|x': src,
      'ivt|no_offset_delta|lead_hours': np.arange(0, 25, 6),
      'ivt|no_offset_delta|want': np.array(
          [[1, nan, nan], [6, 3, nan], [11, 8, 5], [16, 13, 10],
           [nan, 18, 15], [nan, nan, 20]]),
      'ivt|no_offset_delta|want_time_hours': np.arange(0, 61, 12),
      'ivt|no_offset_delta|want_other_hours': np.array([0, 12, 24]),
      'ivt|no_offset_init|x': src,
      'ivt|no_offset_init|lead_hours': np.arange(0, 25, 6),
      'ivt|no_offset_init|want': np.array(
          [[1, 2, 3, 4, 5, nan, nan, nan, nan, nan, nan],
           [nan, nan, 6, 7, 8, 9, 10, nan, nan, nan, nan],
           [nan, nan, nan, nan, 11, 12, 13, 14, 15, nan, nan],
           [nan, nan, nan, nan, nan, nan, 16, 17, 18, 19, 20]]),
      'ivt|no_offset_init|want_time_hours': np.arange(0, 61, 6),
      'ivt|no_offset_init|want_other_hours': np.arange(0, 37, 12),
      'ivt|offset_delta|x': src[:, 1:],
      'ivt|offset_delta|lead_hours': np.arange(6, 25, 6),
      'ivt|offset_delta|want': np.array(
          [[3, nan], [8, 5], [13, 10], [18, 15], [nan, 20]]),
      'ivt|offset_delta|want_time_hours': np.arange(12, 61, 12),
      'ivt|offset_delta|want_other_hours': np.array([12, 24]),
      'ivt|offset_init|x': src[:, 1:],
      'ivt|offset_init|lead_hours': np.arange(6, 25, 6),
      'ivt|offset_init|want': np.array(
          [[2, 3, 4, 5, nan, nan, nan, nan, nan, nan],
           [nan, nan, 7, 8, 9, 10, nan, nan, nan, nan],
           [nan, nan, nan, nan, 12, 13, 14, 15, nan, nan],
           [nan, nan, nan, nan, nan, nan, 17, 18, 19, 20]]),
      'ivt|offset_init|want_time_hours': np.arange(6, 61, 6),
      'ivt|offset_init|want_other_hours': np.arange(0, 37, 12),
  }
  rs = np.random.RandomState(0)
  hours, doys = np.arange(0, 24, 6), np.arange(1, 367)
  clim = rs.normal(size=(hours.size, doys.size, 2, 3, 2))
  times = pd.date_range('2019-12-01', '2020-03-30', freq='6h')
  want = np.stack([clim[np.flatnonzero(hours == t.hour)[0],
                        np.flatnonzero(doys == t.dayofyear)[0]]
                   for t in times])
  out.update({'expand|clim': clim, 'expand|want': want,
              'expand|time_ns': times.values.astype('datetime64[ns]').view(np.int64)})
  return out


def main():
  if len(sys.argv) > 2:  # child: one script per process
    reference, which, path = sys.argv[1], sys.argv[2], sys.argv[3]
    sys.path[:0] = [ROOT, os.path.join(HERE, 'xarray_shim'), reference]
    res = run_probabilistic(reference) if which == 'prob' else run_valid_time(
        reference)
    np.savez(path, **res)
    return
  reference = os.path.abspath(sys.argv[1])
  out = reference_test_arrays()
  import tempfile  # pylint: disable=import-outside-toplevel
  with tempfile.TemporaryDirectory() as tmp:
    for which in ('prob', 'valid'):
      path = os.path.join(tmp, which + '.npz')
      subprocess.run([sys.executable, os.path.abspath(__file__), reference,
                      which, path], check=True)
      with np.load(path) as z:
        out.update({k: z[k] for k in z.files})
  np.savez_compressed(OUT, **out)
  print('wrote', OUT, len(out), 'arrays')


if __name__ == '__main__':
  main()

"""The rule that sends the streamed operators' NumPy input to the `*_host`
entries (weatherbench2_b200/_streamed.py), on the NumPy stand-ins of the
entries, for each family: quantiles, averages, time resampling, precipitation
accumulation, and the mean and quantile climatologies.

  * input already in the entry's layout and dtype reaches the entry in place,
    with no host copy;
  * the streaming budget is the module constant's value when the operator is
    called, so that a caller (or a test forcing many bands) can change it;
  * a climatology variable without cells gives empty float32 results without
    calling the entry."""
import inspect

import numpy as np
import pandas as pd
import pytest

import fake_ctx_average
import fake_ctx_climatology
import fake_ctx_climatology_quantile
import fake_ctx_precip
import fake_ctx_quantile
import fake_ctx_resample
from test_climatology_cpu import _times, make_obs
from weatherbench2_b200 import _derived_precip
from weatherbench2_b200 import preprocessing as pp
from weatherbench2_b200 import resampling
from weatherbench2_b200 import utils
from weatherbench2_b200 import xarray_lite as xl

YEARS = slice('2019', '2020')


def _field(shape):
  return np.random.RandomState(0).standard_normal(shape).astype(np.float32)


def _quantile():
  x = _field((4, 6, 5))
  ds = xl.Dataset({'t': (('time', 'lat', 'lon'), x)})
  return x, lambda: pp.compute_quantiles_core(ds, [0.25, 0.5], 'lat')


def _average():
  x = _field((4, 6, 5))
  ds = xl.Dataset({'t': (('time', 'latitude', 'longitude'), x)})
  return x, lambda: pp.moment_reduce(ds, 'first')


def _resample():
  x = _field((6, 3))
  ds = xl.Dataset({'t': (('time', 'lat'), x)},
                  {'time': pd.date_range('2020-01-01', periods=6).values})
  return x, lambda: resampling.resample_in_time_core(ds, 'resample', '2D',
                                                     'mean', False)


def _precip():
  lead = 'prediction_timedelta'
  x = np.cumsum(np.abs(_field((2, 5))), axis=1, dtype=np.float32)
  ds = xl.Dataset({'tp': (('time', lead), x)},
                  {lead: np.arange(5) * np.timedelta64(6, 'h')})
  op = _derived_precip.PrecipitationAccumulation('tp', 12, lead)
  return x, lambda: op.compute(ds)


def _climatology():
  ds, _, _ = make_obs(layout='3d')
  return ds['z'].data, lambda: utils.compute_hourly_stat(ds, 61, YEARS, 6)


def _climatology_quantile():
  ds, _, _ = make_obs(layout='3d')
  fn = utils.Quantile([0.5]).compute
  return ds['z'].data, lambda: utils.compute_hourly_stat(ds, 61, YEARS, 6, fn)


# family: (its stand-in context, entry, module and name of its budget, case)
FAMILIES = {
    'quantile': (fake_ctx_quantile, 'quantile',
                 (pp, 'QUANTILE_STREAM_BUDGET_BYTES'), _quantile),
    'average': (fake_ctx_average, 'average',
                (pp, 'AVERAGE_STREAM_BUDGET_BYTES'), _average),
    'resample': (fake_ctx_resample, 'time_window_stats',
                 (resampling, 'STREAM_BUDGET_BYTES'), _resample),
    'precip': (fake_ctx_precip, 'precip_accumulation',
               (resampling, 'STREAM_BUDGET_BYTES'), _precip),
    'climatology': (fake_ctx_climatology, 'climatology',
                    (utils, 'STREAM_BUDGET_BYTES'), _climatology),
    'climatology_quantile': (fake_ctx_climatology_quantile,
                             'climatology_quantile',
                             (utils, 'STREAM_BUDGET_BYTES'),
                             _climatology_quantile),
}


def _host_calls(family):
  """Runs the family's case on its stand-in context; the arguments of every
  call of the host entry, by parameter name."""
  fakes, entry, _, case = FAMILIES[family]
  x, run = case()
  calls = []
  with fakes.installed() as fake:
    method = getattr(fake, entry + '_host')
    sig = inspect.signature(method)

    def spy(*args, **kwargs):
      calls.append(sig.bind(*args, **kwargs).arguments)
      return method(*args, **kwargs)

    setattr(fake, entry + '_host', spy)
    run()
  return x, calls


@pytest.mark.parametrize('family', FAMILIES)
def test_host_entry_reads_the_input_in_place(family):
  x, calls = _host_calls(family)
  assert x.dtype == np.float32 and x.flags.c_contiguous
  assert [c['x'] for c in calls] == [x.ctypes.data]


@pytest.mark.parametrize('family', FAMILIES)
def test_host_entry_gets_the_budget_at_call_time(family, monkeypatch):
  module, name = FAMILIES[family][2]
  monkeypatch.setattr(module, name, 3 << 20)
  _, calls = _host_calls(family)
  assert [c['budget'] for c in calls] == [3 << 20]


@pytest.mark.parametrize('quantiles', [None, [0.25, 0.75]])
def test_a_climatology_without_cells_calls_no_entry(quantiles):
  t = _times('2019-01-01', '2021-01-01', 6)
  ds = xl.Dataset({'z': (('time', 'latitude'), np.zeros((t.size, 0),
                                                         np.float32))},
                  {'time': t})
  fakes = fake_ctx_climatology_quantile  # the mean entries too
  with fakes.installed() as fake:
    if quantiles is None:
      out = utils.compute_hourly_stat(ds, 61, YEARS, 6)
      daily = utils.compute_daily_stat(ds, 61, YEARS)
      shape, dshape = (4, 366, 0), (366, 0)
    else:
      fn = utils.Quantile(quantiles).compute
      out = utils.compute_hourly_stat(ds, 61, YEARS, 6, fn)
      daily = utils.compute_daily_stat(ds, 61, YEARS, fn)
      shape, dshape = (4, 2, 366, 0), (2, 366, 0)
  assert fake.calls == []
  for got, want in ((out, shape), (daily, dshape)):
    v = got['z'].values
    assert v.dtype == np.float32 and v.shape == want

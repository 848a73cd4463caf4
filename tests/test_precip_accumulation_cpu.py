"""CPU tests of the precipitation accumulations
(weatherbench2/derived_variables.py:471-528, 685-720): tests/precip_oracle.py
pinned to the reference test's known answers, to vectors made by running the
reference's own classes (tests/golden/reference_precip_vectors.npz, within the
documented float32 bound) and to hand-derived NaN / Inf / clamp / window
cases; then both classes end to end on a NumPy interpretation of the C entry
(tests/fake_ctx_precip.py), with every error they raise."""
import os

import numpy as np
import pytest

import fake_ctx_precip
import precip_oracle as po

HERE = os.path.dirname(os.path.abspath(__file__))
LEAD = 'prediction_timedelta'
NAN = np.nan
INF = np.inf


def _same(got, want):
  got, want = np.asarray(got), np.asarray(want)
  assert got.dtype == want.dtype, (got.dtype, want.dtype)
  np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
  ok = np.isnan(want) | (got == want)
  assert ok.all(), (got, want)
  # -0.0 and +0.0 are told apart
  np.testing.assert_array_equal(np.signbit(got[~np.isnan(want)]),
                                np.signbit(want[~np.isnan(want)]))


def _lead(hours):
  return np.asarray(hours).astype('timedelta64[h]').astype('timedelta64[ns]')


def _ds(x, dims=('time', LEAD), step_hours=6, name='total_precipitation',
        lead=None):
  from weatherbench2_b200 import xarray_lite as xl
  x = np.asarray(x)
  n = x.shape[dims.index(LEAD)] if LEAD in dims else x.shape[-1]
  coords = {LEAD: _lead(np.arange(n) * step_hours) if lead is None else lead}
  if LEAD not in dims:  # a lead coordinate along another dimension
    coords[LEAD] = xl.Coord((dims[-1],), coords[LEAD])
  for d, s in zip(dims, x.shape):
    if d != LEAD:
      coords[d] = np.arange(s)
  return xl.Dataset({name: (dims, x)}, coords)


# ---- the oracle ---------------------------------------------------------------

def test_oracle_reproduces_the_reference_known_answers():
  """derived_variables_test.py:121-216."""
  tp = np.array([0, 5, 15, 14, 20, 30, 30], np.float32)
  _same(po.accumulate(tp, 1), np.array([NAN, 5, 10, 0, 6, 10, 0], np.float32))
  _same(po.accumulate(tp, 4),
        np.array([NAN, NAN, NAN, NAN, 20, 25, 15], np.float32))
  import resample_oracle as ro
  acc = np.array([5, 0, 2, 1, 0, 10], np.float32)
  got = ro.rolling(acc[None], 4, ['sum'], axis=1)['sum'][0]
  np.testing.assert_array_equal(got, [NAN, NAN, NAN, 8, 3, 13])


def _vectors():
  z = np.load(os.path.join(HERE, 'golden', 'reference_precip_vectors.npz'))
  names = sorted({k.split('|')[0] for k in z.files})
  return z, names


def _golden_var(name):
  from weatherbench2_b200 import derived_variables as dv
  return {
      'tp6_w1': dv.PrecipitationAccumulation('total_precipitation', 6),
      'tp24_w4': dv.PrecipitationAccumulation('total_precipitation', 24),
      'tp24_hourly_lead_last': dv.PrecipitationAccumulation(
          'total_precipitation', 24),
      'tp12_noclamp': dv.PrecipitationAccumulation(
          'total_precipitation', 12, set_negative_to_zero=False),
      'agg24_from_6': dv.AggregatePrecipitationAccumulation(24),
  }[name]


def test_oracle_and_operators_match_the_reference_run_vectors():
  z, names = _vectors()
  assert len(names) == 5
  for name in names:
    x, dims = z[f'{name}|x'], tuple(z[f'{name}|dims'])
    want = z[f'{name}|result']
    var = _golden_var(name)
    ax = dims.index(LEAD)
    if name.startswith('agg'):
      import resample_oracle as ro
      xm = np.moveaxis(x, ax, 0)
      mine = np.moveaxis(ro.rolling(xm.reshape(1, xm.shape[0], -1), 4, ['sum'],
                                    axis=1)['sum'].reshape(xm.shape), 0,
                         ax).astype(x.dtype)
      bound = 5 * 2.0**-24 * np.abs(want)
      ds = _ds(x, dims, name='total_precipitation_6hr')
    else:
      w = var.window(_lead(z[f'{name}|lead_hours']))
      mine = po.accumulate(x, w, var.set_negative_to_zero, axis=ax)
      bound = po.reference_bound(x, w, axis=ax)
      ds = _ds(x, dims, lead=_lead(z[f'{name}|lead_hours']))
    assert mine.dtype == want.dtype == np.float32, name
    np.testing.assert_array_equal(np.isnan(mine), np.isnan(want), err_msg=name)
    fin = ~np.isnan(want)
    err = np.abs(mine[fin].astype(np.float64) - want[fin])
    assert (err <= bound[fin]).all(), name
    with fake_ctx_precip.installed():
      got = var.compute(ds)
    assert got.dims == dims, name
    _same(got.values, mine)


def test_nan_and_inf_inside_and_at_each_window_end():
  # w = 3: output t sums x[t] - x[t-3]'s three steps, reading x[t-3 .. t]
  base = np.arange(10, dtype=np.float64) * 2
  for pos in (3, 4, 6):  # oldest value of output 6's window, interior, newest
    for bad in (NAN, INF, -INF):
      x = base.copy()
      x[pos] = bad
      got = po.accumulate(x, 3, clamp=False)
      assert np.isnan(got[:3]).all()
      for t in range(3, 10):
        touches = t - 3 <= pos <= t
        if not touches:
          assert got[t] == 6, (pos, bad, t)
        elif np.isnan(bad) or t - 3 < pos < t:
          # NaN, or an Inf step in and out of the window: inf + -inf
          assert np.isnan(got[t]), (pos, bad, t)
        else:
          # an Inf at one end enters one difference only
          want = bad if pos == t else -bad
          assert got[t] == want, (pos, bad, t)
  # with the clamp, -inf becomes 0 and NaN stays
  x = base.copy()
  x[9] = -INF
  got = po.accumulate(x, 3)
  assert got[9] == 0 and not np.signbit(got[9])
  x[9] = NAN
  assert np.isnan(po.accumulate(x, 3)[9])


def test_negative_steps_clamped_or_kept():
  x = np.array([0, 3, 1, 1, 4, 2], np.float32)
  _same(po.accumulate(x, 1), np.array([NAN, 3, 0, 0, 3, 0], np.float32))
  _same(po.accumulate(x, 1, clamp=False),
        np.array([NAN, 3, -2, 0, 3, -2], np.float32))
  _same(po.accumulate(x, 2), np.array([NAN, NAN, 1, 0, 3, 1], np.float32))
  # -0.0: a sum of one difference -0.0 keeps its sign
  x = np.array([-0.0, 0.0, -0.0], np.float32)
  got = po.accumulate(x, 1)
  assert got[2] == 0 and np.signbit(got[2])  # -0.0 - 0.0 = -0.0


def test_window_one_last_and_longer_than_the_series():
  x = np.cumsum(np.arange(1, 8, dtype=np.float32))
  n = x.size
  _same(po.accumulate(x, 1)[1:], np.diff(x))
  last = po.accumulate(x, n - 1)
  assert np.isnan(last[:-1]).all() and last[-1] == x[-1] - x[0]
  for w in (n, n + 1, 5000):
    assert np.isnan(po.accumulate(x, w)).all()


def test_summed_oldest_first_in_float64():
  x = np.array([0, 2.0**60, 0, 1], np.float32)
  assert po.accumulate(x, 3)[3] == 1  # newest first would give 0
  x = np.array([0, 2.0**60, 0, 1], np.float64)
  assert po.accumulate(x, 3)[3] == 1


@pytest.mark.parametrize('dims', [(LEAD, 'a', 'b'), ('a', LEAD, 'b'),
                                  ('a', 'b', LEAD)])
def test_lead_dimension_first_middle_last(dims):
  from weatherbench2_b200 import derived_variables as dv
  rs = np.random.RandomState(3)
  sizes = {LEAD: 9, 'a': 3, 'b': 4}
  shape = tuple(sizes[d] for d in dims)
  x = np.cumsum(rs.normal(1, 2, size=shape), axis=dims.index(LEAD)).astype(
      np.float32)
  ds = _ds(x, dims)
  with fake_ctx_precip.installed() as fake:
    got = dv.PrecipitationAccumulation('total_precipitation', 12).compute(ds)
  assert got.dims == dims
  ax = dims.index(LEAD)
  _same(got.values, po.accumulate(x, 2, axis=ax))
  # and the series handed to the entry is [outer][lead][inner] in place
  name, nouter, ntime, ninner = fake.calls[-1][:4]
  assert name == 'precip_accumulation_host'
  assert (nouter, ntime, ninner) == (int(np.prod(shape[:ax])), 9,
                                     int(np.prod(shape[ax + 1:])))
  for d in dims:
    np.testing.assert_array_equal(got.coords[d].values, ds.coords[d].values)


def test_dictionary_entries_and_fields():
  from weatherbench2_b200 import derived_variables as dv
  d = dv.DERIVED_VARIABLE_DICT
  p6, p24 = d['total_precipitation_6hr'], d['total_precipitation_24hr']
  assert isinstance(p6, dv.PrecipitationAccumulation)
  assert (p6.accumulation_hours, p24.accumulation_hours) == (6, 24)
  assert p6.total_precipitation_name == 'total_precipitation'
  assert p6.lead_time_name == LEAD and p6.set_negative_to_zero
  assert p6.base_variables == ['total_precipitation']
  assert p6.core_dims == (([LEAD],), [LEAD])
  a6, a12 = (d['total_precipitation_24hr_from_6hr'],
             d['total_precipitation_24hr_from_12hr'])
  assert isinstance(a6, dv.AggregatePrecipitationAccumulation)
  assert (a6.raw_accumulation_name, a6.raw_accumulation_hours) == (
      'total_precipitation_6hr', 6)
  assert (a12.raw_accumulation_name, a12.raw_accumulation_hours) == (
      'total_precipitation_12hr', 12)
  assert a12.base_variables == ['total_precipitation_12hr']
  assert a12.core_dims == (([LEAD],), [LEAD])
  agg = dv.AggregatePrecipitationAccumulation(48)
  assert agg.lead_time_name == LEAD and agg.raw_accumulation_hours == 6


def test_both_classes_end_to_end_float64_and_aggregate():
  from weatherbench2_b200 import derived_variables as dv
  rs = np.random.RandomState(5)
  x = np.cumsum(rs.exponential(1e-3, size=(2, 11, 3)), axis=1)
  ds = _ds(x, ('time', LEAD, 'cell'))
  with fake_ctx_precip.installed():
    got = dv.DERIVED_VARIABLE_DICT['total_precipitation_24hr'].compute(ds)
    assert got.values.dtype == np.float64
    _same(got.values, po.accumulate(x, 4, axis=1))
    six = dv.DERIVED_VARIABLE_DICT['total_precipitation_6hr'].compute(ds)
    ds['total_precipitation_6hr'] = six
    agg = dv.DERIVED_VARIABLE_DICT['total_precipitation_24hr_from_6hr'].compute(
        ds)
  import resample_oracle as ro
  want = ro.rolling(six.values, 4, ['sum'], axis=1)['sum']
  np.testing.assert_array_equal(agg.values, want)
  assert np.isnan(agg.values[:, :4]).all()  # NaN head of w-1, plus the 6 h one


def test_errors():
  from weatherbench2_b200 import derived_variables as dv
  var = dv.PrecipitationAccumulation('total_precipitation', 24)
  x = np.arange(12, dtype=np.float32).reshape(2, 6)
  with fake_ctx_precip.installed():
    with pytest.raises(AssertionError, match='All time steps must be equal.'):
      var.compute(_ds(x, lead=_lead([0, 6, 12, 18, 30, 36])))
    with pytest.raises(AssertionError,
                       match='Accumulation time must be multiple of timestep.'):
      var.compute(_ds(x, step_hours=5))
    with pytest.raises(ValueError, match='at least 2'):
      var.compute(_ds(x[:, :1]))
    with pytest.raises(ValueError, match='positive'):
      var.compute(_ds(x, lead=_lead([36, 30, 24, 18, 12, 6])))
    with pytest.raises(ValueError, match='positive'):
      var.compute(_ds(x, lead=_lead([0] * 6)))
    with pytest.raises(ValueError, match='window of 0'):
      dv.PrecipitationAccumulation('total_precipitation', 0).compute(_ds(x))
    with pytest.raises(ValueError, match='dimension'):
      var.compute(_ds(x, dims=('time', 'step')))
    with pytest.raises(TypeError, match='total_precipitation'):
      var.compute(_ds(x.astype(np.float16)))
    with pytest.raises(TypeError, match='total_precipitation'):
      var.compute(_ds(x.astype(np.int32)))
    with pytest.raises(KeyError):
      var.compute(_ds(x, name='tp'))
    agg = dv.AggregatePrecipitationAccumulation(20)
    acc = _ds(x, name='total_precipitation_6hr')
    with pytest.raises(AssertionError,
                       match='Accumulation time must be multiple of timestep.'):
      agg.compute(acc)
    with pytest.raises(ValueError, match='window of 0'):
      dv.AggregatePrecipitationAccumulation(0).compute(acc)
    with pytest.raises(ValueError, match='dimension'):
      dv.AggregatePrecipitationAccumulation(24).compute(
          _ds(x, dims=('time', 'step'), name='total_precipitation_6hr'))
    with pytest.raises(TypeError, match='total_precipitation_6hr'):
      dv.AggregatePrecipitationAccumulation(24).compute(
          _ds(x.astype(np.int32), name='total_precipitation_6hr'))
    # the window cap of the entry, and a wide window over a short series
    long = _ds(np.zeros((1, 1100), np.float32), step_hours=1)
    with pytest.raises(Exception, match='too wide'):
      dv.PrecipitationAccumulation('total_precipitation', 1050).compute(long)
    wide = dv.PrecipitationAccumulation('total_precipitation', 2000).compute(
        long)
    assert np.isnan(wide.values).all()

"""The SEEPS cases of seeps_cases.py hold up without a GPU: each reaches the
edges it claims and every edge is claimed; the reference (the oracle on the
operands in their own dtypes) still equals the reference run's SEEPS vectors;
the model of the kernel's arithmetic equals float32(reference) bit for bit on
every case; a model of the previous kernel (every operand cast to float32, the
matrix in float64, each step rounded before the time mean) differs on every
float64 case and on a stated share of the realistic cells, so bit equality is
a sharp test; SpatialSEEPS.p1 is NumPy's nanmean in the dry fraction's dtype;
the stand-in context follows the entry and the operators look the wet
threshold up label by label."""
import numpy as np
import pandas as pd
import pytest

import fake_ctx
import seeps_cases as sc

CASES = {c.name: c for c in sc.raw_cases()}
LOOKUPS = {c.name: c for c in sc.lookup_cases()}
F64_CASES = ('f64_forecast_near_thresholds', 'f64_truth_near_thresholds',
             'f64_forecast_f32_truth_wet', 'f32_precip_f64_wet',
             'f64_p1_near_bounds')
# least share of the finite realistic cells the previous kernel gets wrong
# (measured: 5.7, 8.6, 30.3, 4.7 and 6.6 %)
OLD_SHARE = {'era5_1p5_f32': 0.04, 'era5_1p5_f32_mean': 0.06,
             'era5_1p5_f64_mean_skipna': 0.25, 'band_025_f32': 0.03,
             'band_025_f64_precip': 0.04}
MIXES = [(sc.F32,) * 4, (sc.F64,) * 4, (sc.F64, sc.F32, sc.F32, sc.F32),
         (sc.F32, sc.F32, sc.F64, sc.F32), (sc.F32, sc.F32, sc.F32, sc.F64)]


def same(a, b):
  """Bit-equal away from NaN, NaN at the same cells."""
  a, b = np.asarray(a), np.asarray(b)
  nan = np.isnan(a)
  return (a.shape == b.shape and np.array_equal(nan, np.isnan(b)) and
          np.array_equal(a[~nan].view(np.int32), b[~nan].view(np.int32)))


@pytest.mark.parametrize('name', sorted(CASES))
def test_case_reaches_its_edges(name):
  case = CASES[name]
  assert case.edges <= sc.EDGES
  assert not case.edges - sc.reached_edges(case), sorted(
      case.edges - sc.reached_edges(case))


def test_every_edge_is_claimed():
  assert set().union(*(c.edges for c in CASES.values())) == sc.EDGES
  assert set().union(*(c.edges for c in LOOKUPS.values())) == sc.LOOKUP_EDGES
  assert {c.name for c in CASES.values()} >= set(sc.REALISTIC_NAMES)


@pytest.mark.parametrize('name', sorted(LOOKUPS))
def test_lookup_case_reaches_its_edges(name):
  case = LOOKUPS[name]
  assert case.edges <= sc.lookup_reached(case)


def test_reference_equals_the_reference_run_vectors():
  """The oracle, with p1 the float32 nanmean of the dry fraction, gives the
  reference run's SpatialSEEPS maps bit for bit and its SEEPS means to the
  last float64 bits; the kernel model gives float32 of those maps."""
  from golden import reference_cases as rc
  import test_reference_run_vectors as rv
  from oracle import wb2_oracle as orc
  x = rc.extra_inputs()
  vt = x['init'][:, None] + x['lead'][None, :]
  stamps = pd.DatetimeIndex(vt.ravel())
  hour = (np.asarray(stamps.hour) // 12).reshape(vt.shape)
  doy = (np.asarray(stamps.dayofyear) - 1).reshape(vt.shape)
  wet = x['thr'][hour, doy]
  p1 = np.nanmean(x['dry'], axis=(0, 1))
  assert p1.dtype == np.float32
  dims = ('init_time', 'lead_time', 'longitude', 'latitude')
  point = orc.seeps_pointwise(x['pf'], x['pt'], wet, wet, p1, min_p1=0.3,
                              max_p1=0.7)
  wd, want = rv.EXTRA_VECTORS['spatial_seeps']
  perm = [dims.index(d) for d in wd]
  got = np.transpose(point, perm)
  np.testing.assert_array_equal(got, want)
  nf = x['pf'].shape[0] * x['pf'].shape[1]
  case = sc.Case('reference_run', frozenset(), x['pf'].reshape((nf,) + p1.shape),
                 x['pt'].reshape((nf,) + p1.shape), wet.reshape(
                     (nf,) + p1.shape), p1, np.arange(nf), np.arange(nf),
                 min_p1=0.3, max_p1=0.7)
  model = np.transpose(sc.kernel_model(case).reshape(point.shape), perm)
  assert same(model, want.astype(np.float32))
  point = orc.seeps_pointwise(x['pf'], x['pt'], wet, wet, p1)
  got, gd = orc.spatial_average(point, dims, rc.LAT, rc.LON, None, True)
  wd, want = rv.EXTRA_VECTORS['seeps']
  np.testing.assert_allclose(np.transpose(got, [gd.index(d) for d in wd]),
                             want, rtol=1e-15)


@pytest.mark.parametrize('name', sorted(CASES))
def test_kernel_model_equals_float32_reference(name):
  case = CASES[name]
  want = sc.reference(case)
  assert want.shape == (case.nout, case.nrow, case.ncol)
  assert same(sc.kernel_model(case), want)


def _old_share(case):
  want = sc.reference(case)
  old = sc.old_kernel_model(case)
  fin = ~np.isnan(want)
  wrong = ~same_cells(old, want)
  return wrong[fin].mean(), wrong


def same_cells(a, b):
  return (a == b) | (np.isnan(a) & np.isnan(b))


@pytest.mark.parametrize('name', F64_CASES)
def test_previous_kernel_fails_every_float64_case(name):
  share, _ = _old_share(CASES[name])
  assert share > 0


@pytest.mark.parametrize('name', sorted(OLD_SHARE))
def test_previous_kernel_share_on_realistic_cells(name):
  """The previous kernel differs from float32(reference) on a share of the
  realistic cells: rounding the float64 matrix entry once is not the
  reference's float32 chain, and float64 operands were cast to float32."""
  share, _ = _old_share(CASES[name])
  print(f'{name}: previous kernel differs on {100 * share:.2f} % of the '
        'finite cells')
  assert share >= OLD_SHARE[name]


@pytest.mark.parametrize('dtype', [np.float32, np.float64])
def test_p1_is_nanmean_in_the_dry_fraction_dtype(dtype):
  from weatherbench2_b200 import metrics
  case = LOOKUPS['leap_year_6hourly']
  arrays, coords = sc.lookup_data(case, (sc.F32, sc.F32, sc.F32,
                                         np.dtype(dtype)))
  _, _, clim = sc.lookup_datasets(case, arrays, coords)
  p1 = metrics.SpatialSEEPS(climatology=clim).p1
  with np.errstate(all='ignore'):
    import warnings
    with warnings.catch_warnings():
      warnings.simplefilter('ignore', RuntimeWarning)
      want = np.nanmean(arrays['frac'], axis=(0, 1))
  assert p1.dims == ('latitude', 'longitude')
  assert np.asarray(p1.values).dtype == dtype
  np.testing.assert_array_equal(np.asarray(p1.values), want)


@pytest.mark.parametrize('name', sorted(CASES))
def test_fake_context_follows_the_entry(name):
  """The stand-in reads the operands in their own dtypes at the offsets the
  entry takes and agrees with the kernel model bit for bit."""
  case = CASES[name]
  ctx = fake_ctx.FakeContext()
  got = sc.run_entry(ctx, case, ctx.to_device)
  assert same(got, sc.kernel_model(case))


def _operator_maps(case, arrays, coords, op, **kw):
  from weatherbench2_b200 import metrics
  fds, tds, clim = sc.lookup_datasets(case, arrays, coords)
  with fake_ctx.installed():
    m = metrics.SpatialSEEPS(climatology=clim)
    res = getattr(m, op)(fds, tds, **kw)[sc.NAME]
  return np.asarray(res.values), res.dims


@pytest.mark.parametrize('mix', range(len(MIXES)))
@pytest.mark.parametrize('name', sorted(n for n in LOOKUPS
                                        if not LOOKUPS[n].raises))
def test_operator_lookup_on_the_stand_in(name, mix):
  """compute_chunk and the fused time mean through the host code: the wet
  threshold of each valid time found by label, each operand in its dtype."""
  from oracle import wb2_oracle as orc
  case = LOOKUPS[name]
  arrays, coords = sc.lookup_data(case, MIXES[mix], seed=mix)
  dims = ('init_time', 'lead_time', 'latitude', 'longitude')
  got, gd = _operator_maps(case, arrays, coords, 'compute_chunk')
  want = sc.lookup_reference(case, arrays)
  a, b, _ = orc.align(got, gd, want.astype(np.float32), dims)
  assert same(a, b)
  for skipna in (False, True):
    got, gd = _operator_maps(case, arrays, coords, 'compute', skipna=skipna)
    want = sc.lookup_reference(case, arrays, skipna)
    a, b, _ = orc.align(got, gd, want.astype(np.float32), dims[1:])
    assert same(a, b)


def test_missing_valid_hour_raises_key_error():
  case = LOOKUPS['missing_hour']
  arrays, coords = sc.lookup_data(case)
  with pytest.raises(KeyError):
    sc.lookup_positions(case)
  with pytest.raises(KeyError):
    _operator_maps(case, arrays, coords, 'compute_chunk')


@pytest.mark.parametrize('bad', ['f', 't', 'wet', 'frac'])
def test_operands_other_than_float32_or_float64_are_refused(bad):
  case = LOOKUPS['non_leap_daily']
  arrays, coords = sc.lookup_data(case)
  arrays[bad] = arrays[bad].astype(np.float16)
  with pytest.raises(TypeError):
    _operator_maps(case, arrays, coords, 'compute_chunk')

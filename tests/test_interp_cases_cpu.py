"""The interpolation cases of interp_cases.py hold up without a GPU: each
reaches the jnp.interp branches it claims, the host's taps fed through the
kernel's arithmetic equal the float32 jnp.interp model, the model stays within
its float64 bound, mutant lerps differ from the model on a stated share of the
realistic cells (so bit equality is a sharp test), and the transcription of
scipy's linear interp1d equals the installed scipy bit for bit."""
import numpy as np
import pytest

import interp_cases as ic

CASES = {c.name: c for c in ic.bilinear_cases()}
SPECTRA = {c.name: c for c in ic.spectrum_cases()}

# least share of the finite realistic cells where a mutant differs from the
# model: (fused lerp, longitude first)
MUTANT_SHARE = {'upsample_15_to_025': (0.10, 0.20),
                'era5_025_to_64x32': (0.04, 0.12),
                'half_cell_shift': (0.0, 0.20)}


def _same(a, b):
  """Bit-equal away from NaN, NaN at the same cells."""
  nan = np.isnan(a)
  return (np.array_equal(nan, np.isnan(b)) and
          np.array_equal(a[~nan].view(np.int32), b[~nan].view(np.int32)))


def _taps(case):
  from weatherbench2_b200 import regridding  # noqa: F401  (defines Regridder first)
  from weatherbench2_b200 import _regrid_interp as ri
  return ri.BilinearRegridder(case.src.grid(), case.tgt.grid())._taps  # pylint: disable=protected-access


@pytest.mark.parametrize('name', sorted(CASES))
def test_case_reaches_its_branches(name):
  case = CASES[name]
  lat, lon = ic.reached_branches(case)
  assert case.lat_branches <= lat, (sorted(case.lat_branches), sorted(lat))
  assert case.lon_branches <= lon, (sorted(case.lon_branches), sorted(lon))


def test_every_branch_is_reached():
  lat = set().union(*(c.lat_branches for c in CASES.values()))
  lon = set().union(*(c.lon_branches for c in CASES.values()))
  assert {'lerp', 'node', 'left', 'right', 'dx0'} <= lat
  assert {'lerp', 'node', 'left', 'right', 'dx0', 'wrap', 'one_lon'} <= lon
  kinds = {(c.src.periodic, c.src.includes_poles) for c in CASES.values()}
  assert kinds == {(True, True), (True, False), (False, False)}


@pytest.mark.parametrize('name', sorted(CASES))
def test_host_taps_through_kernel_formula_equal_the_model(name):
  case = CASES[name]
  lon, lat = _taps(case)
  got = ic.kernel_formula(case.fields, lon, lat)
  want = ic.bilinear_model(case.fields, case.src, case.tgt)
  assert got.shape == want.shape == (case.fields.shape[0],) + case.tgt.shape
  assert _same(got, want)
  # jnp.interp's `where` returns a clamped or dx0 tap as it is; encoded as a
  # lerp with t = 0 (i1 = i0), an infinite tap would come out NaN
  lerped = [(i0, i1, np.where(t < 0, np.float32(0), t)) for i0, i1, t in
            (lon, lat)]
  old = ic.kernel_formula(case.fields, *lerped)
  if {'left', 'right', 'dx0'} & case.lat_branches and case.src.includes_poles:
    inf = np.isinf(want)
    assert inf.any() and np.isnan(old[inf]).any()


@pytest.mark.parametrize('name', sorted(CASES))
def test_model_within_float64_bound(name):
  case = CASES[name]
  model = ic.bilinear_model(case.fields, case.src, case.tgt)
  ref = ic.bilinear_float64(case.fields, case.src, case.tgt)
  bound = ic.bilinear_bound(case.fields, case.src, case.tgt)
  fin = np.isfinite(ref)
  assert np.array_equal(np.isnan(model), np.isnan(ref))
  assert np.array_equal(model[np.isinf(ref)], ref[np.isinf(ref)])
  assert np.all(np.abs(model[fin] - ref[fin]) <= bound[fin])
  # constants come back exactly
  const = case.fields[case.nreal]
  out = model[case.nreal]
  assert np.all((out == const.flat[0]) | np.isnan(out))


@pytest.mark.parametrize('name', sorted(MUTANT_SHARE))
def test_mutant_lerps_differ_from_the_model(name):
  case = CASES[name]
  real = case.fields[:case.nreal]
  model = ic.bilinear_model(real, case.src, case.tgt)
  fin = np.isfinite(model)
  for mutant, share in zip((ic.bilinear_fma, ic.bilinear_lon_first),
                           MUTANT_SHARE[name]):
    got = mutant(real, case.src, case.tgt)
    assert np.mean(got[fin] != model[fin]) >= share, mutant.__name__
    # rtol = 2e-5, the tolerance these regridders were held to before, sees
    # almost none of it
    seen = ~np.isclose(got[fin], model[fin], rtol=2e-5, atol=2e-6)
    assert np.mean(seen) < 1e-4, mutant.__name__


def test_jnp_remainder_keeps_negative_zero():
  x = np.array([-0.0, -1e-6, 360.0, -360.0, 725.5], np.float32)
  r = ic.jnp_remainder(x, np.float32(360))
  assert np.signbit(r[0]) and r[0] == 0
  np.testing.assert_array_equal(r[1:], np.float32([360.0, 0.0, 0.0, 5.5]))


@pytest.mark.parametrize('name', sorted(SPECTRA))
def test_weighted_form_equals_installed_scipy(name):
  case = SPECTRA[name]
  with np.errstate(invalid='ignore'):
    want = ic.scipy_reference(case)
  got = ic.scipy_weighted(case)
  assert np.array_equal(got.view(np.int64), want.view(np.int64)) or (
      np.array_equal(np.isnan(got), np.isnan(want)) and
      np.array_equal(got[~np.isnan(got)], want[~np.isnan(want)]))
  # the float32 rounding of scipy's value is within the bound of the exact
  # interpolant
  exact = ic.exact_spectrum(case)
  fin = np.isfinite(exact)
  err = np.abs(want.astype(np.float32).astype(np.float64)[fin] -
               exact[fin].astype(np.float64))
  assert np.all(err <= ic.spectrum_bound(case)[fin])


@pytest.mark.parametrize('name', sorted(SPECTRA))
def test_spectrum_cases_reach_nodes_edges_and_non_finite(name):
  case = SPECTRA[name]
  tab, f = case.table, case.freqs
  on_node = np.isin(f, tab[:, 1:-1] if tab.shape[1] > 2 else tab)
  assert on_node.any() and np.isnan(f).any()
  assert (f < tab[:, :1].min()).any() and (f > tab[:, -1:].max()).any()
  if case.table.shape[1] > 4:
    with np.errstate(invalid='ignore'):
      want = ic.scipy_reference(case)
    inside = (f >= tab[:, :1]) & (f <= tab[:, -1:])  # (nrow, nf)
    # inf and NaN spectra reach the output inside the rows' ranges
    assert np.isinf(want[:, inside]).any() and np.isnan(want[:, inside]).any()
    # one float64 ulp outside a row's ends is NaN, at and inside is not
    r = tab.shape[0] // 3
    row = want[0, r]
    for end, sign in ((tab[r, 0], -1), (tab[r, -1], 1)):
      assert np.isnan(row[f == np.nextafter(end, sign * np.inf)]).all()
      assert not np.isnan(row[f == end]).all()


def test_stand_in_spectrum_interp_equals_scipy():
  import fake_ctx
  case = SPECTRA['zonal_240x121']
  spec = np.ascontiguousarray(case.spec)
  out = np.empty(case.spec.shape[:2] + (case.freqs.size,), np.float32)
  fake_ctx.FakeContext().spectrum_interp(
      spec.ctypes.data, case.nfield, *case.table.shape, case.table,
      case.freqs, out.ctypes.data)
  with np.errstate(invalid='ignore'):
    want = ic.scipy_reference(case).astype(np.float32)
  assert _same(out, want)

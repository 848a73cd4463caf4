"""The zonal-spectrum cases of tests/spectrum_cases.py (no GPU): they reach
what they claim, their float64 answers equal the oracle's, and the per-bin
bound separates a float32 transform of the raw row (fails on rows whose mean
is large against their variation) from one of the shifted row (passes, and
not by a slack margin)."""
import numpy as np
import pytest

import spectrum_cases as sc
from oracle import wb2_oracle as orc


@pytest.mark.parametrize('n', [1440, 720, 240])
def test_tones_cover_every_crt_class(n):
  ra, rb, rc = sc.crt_bins(n)
  bins = sc.tone_bins(n)
  assert {(p % ra, p % rb) for p in bins} == {(a, b) for a in range(ra) for b in range(rb)}
  assert {p % rc for p in bins} == set(range(rc))
  assert {1, n // 2 - 1, n // 2} <= set(bins)


@pytest.mark.parametrize('n', [1440, 720, 240])
def test_nonfinite_rows_sit_where_they_claim(n):
  g = sc.PFA_PLANS[n][3]
  nrow, where = sc.nonfinite_rows(n)
  assert nrow % 2 == 1
  assert where['row_a'] % 2 == 0 and where['row_b'] % 2 == 1
  assert (where['first_pair_of_group'] // 2) % g == 0
  assert (where['last_pair_of_group'] // 2) % g == g - 1
  assert where['last_odd_row'] == nrow - 1
  npair, ngroup, _ = sc.pfa_geometry(n, nrow)
  assert npair == (nrow + 1) // 2 and ngroup == 3  # the last group is partial


@pytest.mark.parametrize('n,nrow,nslot,chunks', [
    (1440, 721, 1, 181), (1440, 721, 2, 181), (1440, 721, 37 * 5, 9),
    (1440, 4, 1, 1), (720, 361, 1, 37), (240, 121, 3, 11)])
def test_mode2_chunk_counts(n, nrow, nslot, chunks):
  assert sc.pfa_geometry(n, nrow, nslot)[2] == chunks


def test_paths():
  assert sc.path_for(1440) == 'pfa'
  assert sc.path_for(1440, aligned=False) == 'fixed'
  assert sc.path_for(1440, force='generic') == 'generic'
  assert sc.path_for(512) == 'fixed' and sc.path_for(64) == 'fixed'
  for n in (2, 4, 12, 18, 36):
    assert sc.path_for(n) == 'generic'


@pytest.mark.parametrize('kind', sc.REALISTIC)
def test_reference_equals_oracle(kind):
  nrow, n = 5, 1440
  x = sc.realistic(kind, nrow, n, seed=3)
  lat = np.linspace(-60, 60, nrow)
  lon = np.linspace(0, 360, n, endpoint=False)
  # the oracle on the float32 row widened to float64: NumPy >= 2 runs rfft on
  # float32 input in float32, whose tail is as noisy as a raw float32 FFT's
  spec, _, _, _ = orc.zonal_energy_spectrum(x.astype(np.float64),
                                            ('latitude', 'longitude'), lat, lon)
  np.testing.assert_allclose(sc.want(x, orc.circumference(lat)), spec, rtol=1e-12, atol=0)


@pytest.mark.parametrize('n', [1440, 720, 240, 64, 12, 2])
def test_structural_answers_are_exact(n):
  for name, row, exact in sc.structural(n):
    np.testing.assert_allclose(sc.want(row[None], np.ones(1))[0], exact,
                               rtol=1e-12, atol=1e-20, err_msg=name)


@pytest.mark.parametrize('n', [1440, 720, 240])
@pytest.mark.parametrize('kind', sc.LARGE_MEAN)
def test_bound_fails_raw_and_holds_shifted_in_float32_model(n, kind):
  x = sc.realistic(kind, 6, n, seed=n)
  scale = np.ones(6)
  b, w = sc.bound(x, scale, 'pfa')
  raw = np.abs(sc.pfa_model(x, shift=False) - w) / b
  shifted = np.abs(sc.pfa_model(x, shift=True) - w) / b
  assert raw.max() > 1.0, 'the raw transform must fail the bound'
  assert shifted.max() <= 1.0
  if n == 1440:
    assert shifted[:, 1:].max() >= 0.1, 'the bound is slack away from bin 0'


@pytest.mark.parametrize('n', [1440, 720, 240])
def test_float32_model_of_pfa_plan_is_the_dft(n):
  x = sc.realistic('white', 3, n, seed=1)
  np.testing.assert_allclose(sc.pfa_model(x, shift=True), sc.want(x, np.ones(3)),
                             rtol=1e-4, atol=1e-9)

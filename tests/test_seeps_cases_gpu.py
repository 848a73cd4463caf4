"""K9 (csrc/seeps.cu) on the seeded cases of seeps_cases.py.

The raw entry must give float32 of the reference bit for bit on every case,
NaN pattern included, and the same bits on a second call.  The reference is
the oracle on the operands in their own dtypes followed by Metric.compute's
float64 time mean: one comparison in the wrong precision moves a cell to
another category, so nothing here is compared with a tolerance except the
spatial means.  The operators (SpatialSEEPS.compute_chunk, SpatialSEEPS.compute
with skipna both ways, SEEPS.compute_chunk over the official regions) run on
NumPy and on CUDA input, float32 and float64, with valid times on Feb 29 and
across the year boundary against a 6-hourly climatology: the maps must equal
the reference bit for bit, the spatial means stay within the K1 realistic
bound of test_region_reduce_gpu.py."""
import numpy as np
import pytest

import seeps_cases as sc

pytestmark = pytest.mark.gpu

CASES = {c.name: c for c in sc.raw_cases()}
U = 2.0 ** -24


@pytest.fixture(scope='module')
def ctx():
  from weatherbench2_b200 import _lib
  return _lib.default_context(0)


def same(a, b):
  a, b = np.asarray(a), np.asarray(b)
  nan = np.isnan(a)
  return (a.shape == b.shape and np.array_equal(nan, np.isnan(b)) and
          np.array_equal(a[~nan].view(np.int32), b[~nan].view(np.int32)))


def _first_diff(a, b):
  bad = np.argwhere(~((a == b) | (np.isnan(a) & np.isnan(b))))[:5]
  return [(tuple(i), a[tuple(i)], b[tuple(i)]) for i in bad]


@pytest.mark.parametrize('name', sorted(CASES))
def test_raw_entry_equals_the_reference(ctx, name):
  import torch
  case = CASES[name]
  keep = []

  def upload(a):
    keep.append(torch.from_numpy(np.ascontiguousarray(a)).cuda())
    return keep[-1].data_ptr()

  want = sc.reference(case)
  got = sc.run_entry(ctx, case, upload)
  assert same(got, want), _first_diff(got, want)
  again = sc.run_entry(ctx, case, upload)
  assert np.array_equal(again.view(np.int32), got.view(np.int32))


def _np(v):
  return v.cpu().numpy() if hasattr(v, 'cpu') else np.asarray(v)


def _oracle_region(r, lat, lon):
  from oracle import wb2_oracle as orc
  from weatherbench2_b200 import regions as R
  if isinstance(r, R.SliceRegion):
    return orc.SliceRegion(lat_slice=r.lat_slice, lon_slice=r.lon_slice)
  if isinstance(r, R.LandRegion):
    return orc.LandRegion(np.asarray(r.land_sea_mask), r.threshold, lat, lon)
  return orc.CombinedRegion([_oracle_region(x, lat, lon) for x in r.regions])


@pytest.mark.parametrize('on', ['numpy', 'cuda'])
@pytest.mark.parametrize('dtype', [np.float32, np.float64])
def test_operators(on, dtype):
  import torch
  import region_cases as rc
  from oracle import wb2_oracle as orc
  from weatherbench2_b200 import metrics
  case = [c for c in sc.lookup_cases() if c.name == 'leap_year_6hourly'][0]
  dt = np.dtype(dtype)
  arrays, coords = sc.lookup_data(case, (dt,) * 4, nlat=121, nlon=240,
                                  seed=21)
  to = (lambda a: torch.from_numpy(a).cuda()) if on == 'cuda' else None
  fds, tds, clim = sc.lookup_datasets(case, arrays, coords, to)
  dims = ('init_time', 'lead_time', 'latitude', 'longitude')
  want = sc.lookup_reference(case, arrays)
  res = metrics.SpatialSEEPS(climatology=clim).compute_chunk(fds, tds)[sc.NAME]
  a, b, _ = orc.align(_np(res.values), res.dims, want.astype(np.float32), dims)
  assert same(a, b), _first_diff(a, b)
  for skipna in (False, True):
    res = metrics.SpatialSEEPS(climatology=clim).compute(
        fds, tds, skipna=skipna)[sc.NAME]
    mean = sc.lookup_reference(case, arrays, skipna)
    a, b, _ = orc.align(_np(res.values), res.dims, mean.astype(np.float32),
                        dims[1:])
    assert same(a, b), (skipna, _first_diff(a, b))
  # SEEPS: the K1 reduction of the maps with skipna, per official region.
  # The maps are float32(reference) and non-negative, so K1's realistic bound
  # |kernel - ref| <= k u sum |W v| / sum W is k u |ref|, k = ncol + 89
  lat, lon = coords['lat'], coords['lon']
  lsm = rc.fractional_lsm(lat.size, lon.size)
  k = lon.size + 89
  for region in rc.official_regions(lsm):
    res = metrics.SEEPS(climatology=clim).compute_chunk(fds, tds,
                                                        region=region)[sc.NAME]
    ref, rd = orc.spatial_average(want, dims, lat, lon,
                                  _oracle_region(region, lat, lon), True)
    a, b, _ = orc.align(_np(res.values).astype(np.float64), res.dims, ref, rd)
    assert np.array_equal(np.isnan(a), np.isnan(b)), region
    fin = ~np.isnan(b)
    assert (np.abs(a - b)[fin] <= k * U * np.abs(b)[fin]).all(), (
        region, np.abs(a - b)[fin].max(), np.abs(b)[fin].max())

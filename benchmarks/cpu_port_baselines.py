#!/usr/bin/env python
"""Times the oracle port (oracle/wb2_oracle.py, the NumPy restatement of the
reference's xarray / NumPy / JAX op sequence) for every kernel of the hot path
on ONE host core, on bounded samples of the BASELINE shapes, so that each GPU
kernel has the reference's CPU path timed beside it (SURVEY.md section 8d).
One JSON line per path.  `python benchmarks/cpu_port_baselines.py`
"""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import wb2_oracle as orc  # noqa: E402

NLAT, NLON = 721, 1440


def timed(fn, reps=2):
  fn()
  t0 = time.perf_counter()
  for _ in range(reps):
    fn()
  return (time.perf_counter() - t0) / reps


def main():
  rs = np.random.RandomState(0)
  lat = np.linspace(-90, 90, NLAT)
  lon = np.arange(NLON) * 0.25
  out = []
  # K1: RMSE + Bias + ACC on 13 levels x 721 x 1440
  dims = ('level', 'latitude', 'longitude')
  f, t, c = (rs.standard_normal((13, NLAT, NLON)).astype(np.float32)
             for _ in range(3))

  def k1():
    orc.rmse_sqrt_before_time_avg(f, dims, t, dims, lat, lon)
    orc.bias(f, dims, t, dims, lat, lon)
    orc.acc(f, dims, t, dims, c, dims, lat, lon)
  s = timed(k1)
  out.append({'path': 'K1 RMSE+Bias+ACC', 'sample': '13 x 721 x 1440 cells',
              'seconds': s, 'grid_cells_per_s': f.size / s})
  # K2: CRPS + ensemble-mean MSE + variance, M = 50, a 32-row latitude band
  sel = slice(344, 376)
  x = rs.standard_normal((50, 32, NLON)).astype(np.float32)
  tt = rs.standard_normal((32, NLON)).astype(np.float32)
  ed = ('realization', 'latitude', 'longitude')
  td = ('latitude', 'longitude')

  def k2():
    orc.crps(x, ed, tt, td, 'realization', lat[sel], lon)
    orc.ensemble_mean_mse(x, ed, tt, td, 'realization', lat[sel], lon)
    orc.ensemble_variance(x, ed, 'realization', lat[sel], lon)
  s = timed(k2, reps=1)
  out.append({'path': 'K2 CRPS+ens-mean MSE+variance (M=50)',
              'sample': '50 members x 32 x 1440 grid points',
              'seconds': s, 'grid_points_per_s': tt.size / s})

  def k3():
    orc.energy_score(x, ed, tt, td, 'realization', lat[sel], lon)
  s = timed(k3, reps=1)
  out.append({'path': 'K3 energy score (M=50)',
              'sample': '50 members x 32 x 1440 grid points',
              'seconds': s, 'grid_points_per_s': tt.size / s})
  # K5: conservative regrid 0.25 -> 1.5 degrees, 2 fields (dense einsum, as the
  # reference does)
  src = orc.Grid(longitudes=lon, latitudes=lat)
  tgt = orc.Grid(longitudes=np.arange(240) * 1.5,
                 latitudes=np.linspace(-90, 90, 121))
  xr_ = rs.standard_normal((2, NLON, NLAT)).astype(np.float32)
  s = timed(lambda: orc.conservative_regrid(xr_, src, tgt), reps=1)
  out.append({'path': 'K5 conservative regrid 0.25->1.5deg',
              'sample': '2 fields of 1440 x 721', 'seconds': s,
              'source_cells_per_s': xr_.size / s})
  # K4: zonal spectrum of 13 x 721 x 1440
  xs = rs.standard_normal((13, NLAT, NLON)).astype(np.float32)
  s = timed(lambda: orc.zonal_energy_spectrum(xs, dims, lat, lon))
  out.append({'path': 'K4 zonal energy spectrum', 'sample': '13 x 721 x 1440',
              'seconds': s, 'grid_cells_per_s': xs.size / s})
  # climatology: hourly explicit mean + std (compute_climatology.py's default
  # method), 4 years 6-hourly, 64 cells of the 721 x 1440 grid
  sys.path.insert(0, os.path.join(ROOT, 'tests'))
  import climatology_oracle as co  # pylint: disable=import-outside-toplevel
  times = np.arange(np.datetime64('2017-01-01', 'ns'),
                    np.datetime64('2021-01-01', 'ns'), np.timedelta64(6, 'h'))
  xc = rs.standard_normal((times.size, 64)).astype(np.float32)

  def clim():
    for stat in ('mean', 'std'):
      co.hourly_stat(times, xc, 61, slice('2017', '2020'), 6, stat)
  s = timed(clim, reps=1)
  out.append({'path': 'climatology hourly explicit mean+std',
              'sample': f'{times.size} 6-hourly steps x 64 cells',
              'seconds': s, 'values_per_s': xc.size / s})
  for o in out:
    o.update({'cores': 1, 'kind': 'port'})
    print(json.dumps(o), flush=True)


if __name__ == '__main__':
  main()

#!/usr/bin/env python
"""Per-kernel micro-benchmarks (device-resident synthetic inputs, CUDA events
on the launching stream, >= 3 warm-up launches, inputs >> L2).  One JSON line
per kernel with the achieved algorithmic HBM GB/s and the fraction of the
measured peak (MEASURED_PEAKS.json; else the H100 SXM data sheet's 3.35 TB/s).  The
headline contract line is bench.py.

  python benchmarks/bench_kernels.py --kernel ens      # K2, BASELINE configs[2]
  python benchmarks/bench_kernels.py --kernel det      # K1 variants
  python benchmarks/bench_kernels.py --kernel regrid   # K5, configs[3]
  python benchmarks/bench_kernels.py --kernel spectrum # K4, configs[4]
  python benchmarks/bench_kernels.py --kernel climatology --steps 3
  python benchmarks/bench_kernels.py --kernel climatology_quantile --steps 2
  python benchmarks/bench_kernels.py --kernel resample --steps 5
  python benchmarks/bench_kernels.py --kernel wind_dynamics --steps 20
  python benchmarks/bench_kernels.py --kernel precip_accumulation --steps 20
  python benchmarks/bench_kernels.py --kernel column_integral --steps 20
  python benchmarks/bench_kernels.py --kernel quantile --steps 5
  python benchmarks/bench_kernels.py --kernel average --steps 5
  python benchmarks/bench_kernels.py --kernel slab_gather --steps 10
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

NLAT, NLON = 721, 1440


def peak():
  try:
    return float(json.load(open(os.path.join(ROOT, 'MEASURED_PEAKS.json')))[
        'hbm_gbs'])
  except Exception:  # pylint: disable=broad-except
    return 3350.0


def timeit(fn, steps, warmup=3):
  import torch
  for _ in range(warmup):
    fn()
  torch.cuda.synchronize()
  e0 = torch.cuda.Event(enable_timing=True)
  e1 = torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(steps):
    fn()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / steps


def setup():
  import torch
  from weatherbench2_b200 import _lib
  torch.cuda.set_device(0)
  stream = torch.cuda.Stream()
  torch.cuda.set_stream(stream)
  ctx = _lib.Context(0)
  ctx.set_stream(stream.cuda_stream)
  return torch, _lib, ctx


def report(name, ms, nbytes, units, unit_name, extra=None):
  gbs = nbytes / (ms * 1e-3) / 1e9
  line = {'kernel': name, 'ms': ms, 'algorithmic_GB': nbytes / 1e9,
          'achieved_GBps': gbs, 'peak_GBps': peak(), 'frac': gbs / peak(),
          unit_name + '_per_s': units / (ms * 1e-3)}
  line.update(extra or {})
  print(json.dumps(line), flush=True)


def bench_ens(args):
  torch, _lib, ctx = setup()
  from weatherbench2_b200 import _spatial as sp
  lat = np.linspace(-90, 90, NLAT)
  lon = np.arange(NLON) * 0.25
  for m in args.members:
    nfield = args.fields
    x = torch.randn((m, nfield, NLAT, NLON), device='cuda',
                    dtype=torch.float32)
    x += torch.randn((1, nfield, NLAT, NLON), device='cuda')  # shared signal
    t = torch.randn((nfield, NLAT, NLON), device='cuda', dtype=torch.float32)
    (_, spec), = sp.build_weights(ctx, lat, lon, [None], 'lat_lon', NLON)
    slab = NLAT * NLON
    base = min(x.data_ptr(), t.data_ptr())
    off_x = np.arange(nfield, dtype=np.int64) * slab + (x.data_ptr() -
                                                        base) // 4
    off_t = np.arange(nfield, dtype=np.int64) * slab + (t.data_ptr() -
                                                        base) // 4
    out = torch.zeros((nfield, _lib.ENS_NSTAT), device='cuda',
                      dtype=torch.float64)
    for skipna in (False, True):
      fn = lambda: ctx.ens_metrics(base, base, _lib.F32, m, nfield * slab,
                                   off_x, off_t, spec, skipna, out.data_ptr())
      ms = timeit(fn, args.steps)
      pts = nfield * slab
      report(f'ens_metrics M={m} skipna={skipna}', ms, pts * (4 * m + 4), pts,
             'grid_points', {'members': m, 'fields': nfield})
    del x, t


def bench_energy(args):
  torch, _lib, ctx = setup()
  from weatherbench2_b200 import _spatial as sp
  lat = np.linspace(-90, 90, NLAT)
  lon = np.arange(NLON) * 0.25
  for m in args.members:
    nfield = args.fields
    x = torch.randn((m, nfield, NLAT, NLON), device='cuda',
                    dtype=torch.float32)
    t = torch.randn((nfield, NLAT, NLON), device='cuda', dtype=torch.float32)
    (_, spec), = sp.build_weights(ctx, lat, lon, [None], 'lat_lon', NLON)
    slab = NLAT * NLON
    base = min(x.data_ptr(), t.data_ptr())
    off_x = np.arange(nfield, dtype=np.int64) * slab + (x.data_ptr() -
                                                        base) // 4
    off_t = np.arange(nfield, dtype=np.int64) * slab + (t.data_ptr() -
                                                        base) // 4
    out = torch.zeros((nfield, 1, 4, m), device='cuda', dtype=torch.float64)
    fn = lambda: ctx.energy_score(base, base, _lib.F32, m, nfield * slab,
                                  off_x, off_t, spec, out.data_ptr())
    ms = timeit(fn, args.steps)
    pts = nfield * slab
    report(f'energy_score M={m}', ms, pts * (4 * m + 4), pts, 'grid_points',
           {'members': m, 'fields': nfield})
    del x, t


def bench_det(args):
  torch, _lib, ctx = setup()
  from weatherbench2_b200 import _spatial as sp, regions as R
  lat = np.linspace(-90, 90, NLAT)
  lon = np.arange(NLON) * 0.25
  nfield = args.fields
  f = torch.randn((nfield, NLAT, NLON), device='cuda', dtype=torch.float32)
  t = torch.randn_like(f)
  c = torch.randn_like(f)
  slab = NLAT * NLON
  base = min(f.data_ptr(), t.data_ptr(), c.data_ptr())
  offs = [np.arange(nfield, dtype=np.int64) * slab + (v.data_ptr() - base) // 4
          for v in (f, t, c)]
  regs13 = [None, R.SliceRegion(lat_slice=slice(-20, 20)),
            R.ExtraTropicalRegion(),
            R.SliceRegion(lat_slice=slice(20, 90)),
            R.SliceRegion(lat_slice=slice(-90, -20)),
            R.SliceRegion(lat_slice=slice(35, 75),
                          lon_slice=[slice(347.5, None), slice(0, 42.5)]),
            R.SliceRegion(lat_slice=slice(25, 60), lon_slice=slice(240, 290)),
            R.SliceRegion(lat_slice=slice(25, 60), lon_slice=slice(145, 180)),
            R.SliceRegion(lat_slice=slice(25, 60), lon_slice=slice(102.5, 150)),
            R.SliceRegion(lat_slice=slice(-45, -12.5),
                          lon_slice=slice(120, 175)),
            R.SliceRegion(lat_slice=slice(-37.5, -22.5),
                          lon_slice=slice(15, 50)),
            R.SliceRegion(lat_slice=slice(-52.5, -20),
                          lon_slice=slice(287.5, 327.5)),
            R.SliceRegion(lat_slice=slice(-90, -60))]
  cases = [('global', [None]), ('3 lat-band regions', regs13[:3]),
           ('13 regions (lat/lon boxes)', regs13)]
  for label, regs in cases:
    (_, spec), = sp.build_weights(ctx, lat, lon, regs, 'lat_lon', NLON)
    out = torch.zeros((nfield, len(regs), _lib.DET_NSTAT), device='cuda',
                      dtype=torch.float64)
    for clim in (True, False):
      for path in ('tma', 'ldg'):
        os.environ['WB2_DET_PATH'] = path
        fn = lambda: ctx.det_metrics(
            base, base, base if clim else None, _lib.F32, offs[0], offs[1],
            offs[2] if clim else None, spec, False, out.data_ptr())
        ms = timeit(fn, args.steps)
        cells = nfield * slab
        report(f'det_metrics {label} clim={clim} path={path} nseg={spec.nseg}',
               ms, cells * (12 if clim else 8), cells, 'grid_cells')
  os.environ.pop('WB2_DET_PATH', None)


def bench_regrid(args):
  torch, _lib, ctx = setup()
  from weatherbench2_b200 import regridding
  src = regridding.Grid.from_degrees(np.arange(NLON) * 0.25,
                                     np.linspace(-90, 90, NLAT))
  tgt = regridding.Grid.from_degrees(np.arange(240) * 1.5,
                                     np.linspace(-90, 90, 121))
  rg = regridding.ConservativeRegridder(source=src, target=tgt)
  nfield = args.fields
  x = torch.randn((nfield, NLON, NLAT), device='cuda', dtype=torch.float32)
  out = torch.empty((nfield, 240, 121), device='cuda', dtype=torch.float32)
  fn = lambda: rg.regrid_device(ctx, x.data_ptr(), out.data_ptr(), nfield)
  ms = timeit(fn, args.steps)
  cells = nfield * NLAT * NLON
  report('regrid_conservative 0.25->1.5deg', ms,
         cells * 4 + nfield * 240 * 121 * 4, cells, 'source_cells')


def bench_spectrum(args):
  torch, _lib, ctx = setup()
  nfield = args.fields
  x = torch.randn((nfield, NLAT, NLON), device='cuda', dtype=torch.float32)
  nk = NLON // 2 + 1
  scale = np.cos(np.deg2rad(np.linspace(-90, 90, NLAT))) * 4.0e7
  out = torch.empty((nfield, NLAT, nk), device='cuda', dtype=torch.float32)
  fn = lambda: ctx.zonal_spectrum(x.data_ptr(), nfield, NLAT, NLON, scale,
                                  out.data_ptr())
  ms = timeit(fn, args.steps)
  cells = nfield * NLAT * NLON
  report('zonal_spectrum per-time output', ms, cells * 4 + nfield * NLAT * nk *
         4, cells, 'grid_cells')
  acc = torch.zeros((13, NLAT, nk), device='cuda', dtype=torch.float32)
  fn = lambda: ctx.zonal_spectrum(x.data_ptr(), nfield, NLAT, NLON, scale,
                                  acc.data_ptr(), True, 13)
  ms = timeit(fn, args.steps)
  report('zonal_spectrum time-summed output', ms, cells * 4, cells,
         'grid_cells')
  red = torch.zeros((13, nk), device='cuda', dtype=torch.float32)
  fn = lambda: ctx.zonal_spectrum_latsum(x.data_ptr(), nfield, NLAT, NLON,
                                         scale, red.data_ptr(), 13)
  ms = timeit(fn, args.steps)
  report('zonal_spectrum + latitude-weighted reduction (latsum)', ms,
         cells * 4, cells, 'grid_cells')


def bench_maps(args):
  """K6 / K6e: Spatial* maps; per-time maps (ngroup 1) and a 10-step time mean
  fused in (ngroup 10)."""
  torch, _lib, ctx = setup()
  slab = NLAT * NLON
  nfield = 390  # 10 times x 39 (variable, level) maps
  f = torch.randn((nfield, NLAT, NLON), device='cuda', dtype=torch.float32)
  t = torch.randn((nfield, NLAT, NLON), device='cuda', dtype=torch.float32)
  base = min(f.data_ptr(), t.data_ptr())
  for ngroup in (1, 10):
    nout = nfield // ngroup
    # group-major tables: output j averages times g of (variable, level) j
    idx = (np.arange(ngroup)[None, :] * nout + np.arange(nout)[:, None])
    off_f = (idx * slab + (f.data_ptr() - base) // 4).astype(np.int64).ravel()
    off_t = (idx * slab + (t.data_ptr() - base) // 4).astype(np.int64).ravel()
    out = torch.empty((nout, NLAT, NLON), device='cuda', dtype=torch.float32)
    fn = lambda: ctx.det_maps(base, base, _lib.F32, _lib.MAP_MSE, nout, ngroup,
                              off_f, off_t, NLAT, NLON, NLON, False,
                              out.data_ptr())
    ms = timeit(fn, args.steps)
    cells = nfield * slab
    report(f'det_maps MSE ngroup={ngroup}', ms, cells * 8 + nout * slab * 4,
           cells, 'grid_cells')
  del f, t
  for m in args.members:
    ntime, nmap = 5, 8
    x = torch.randn((m, ntime * nmap, NLAT, NLON), device='cuda',
                    dtype=torch.float32)
    t = torch.randn((ntime * nmap, NLAT, NLON), device='cuda',
                    dtype=torch.float32)
    base = min(x.data_ptr(), t.data_ptr())
    for ngroup, mask in ((1, _lib.ENS_CRPS), (ntime, _lib.ENS_CRPS),
                         (ntime, 63)):
      nout = ntime * nmap // ngroup
      idx = (np.arange(ngroup)[None, :] * nout + np.arange(nout)[:, None])
      off_x = (idx * slab + (x.data_ptr() - base) // 4).astype(
          np.int64).ravel()
      off_t = (idx * slab + (t.data_ptr() - base) // 4).astype(
          np.int64).ravel()
      nsel = bin(mask).count('1')
      out = torch.empty((nsel, nout, NLAT, NLON), device='cuda',
                        dtype=torch.float32)
      fn = lambda: ctx.ens_maps(base, base, _lib.F32, m, ntime * nmap * slab,
                                nout, ngroup, off_x, off_t, NLAT, NLON, NLON,
                                mask, False, out.data_ptr())
      ms = timeit(fn, args.steps)
      pts = ntime * nmap * slab
      report(f'ens_maps M={m} ngroup={ngroup} nsel={nsel}', ms,
             pts * (4 * m + 4) + nsel * nout * slab * 4, pts, 'grid_points')
    del x, t


def bench_threshold(args):
  """K7: ensemble Brier / debiased / ignorance / RPS for 4 Gaussian-quantile
  thresholds from one pass, and the Gaussian-forecast entry."""
  torch, _lib, ctx = setup()
  from weatherbench2_b200 import _spatial as sp
  lat = np.linspace(-90, 90, NLAT)
  lon = np.arange(NLON) * 0.25
  (_, spec), = sp.build_weights(ctx, lat, lon, [None], 'lat_lon', NLON)
  slab = NLAT * NLON
  nfield = args.fields
  z = np.array([-1.2816, -0.5244, 0.5244, 1.2816])
  for m in args.members:
    x = torch.randn((m, nfield, NLAT, NLON), device='cuda',
                    dtype=torch.float32)
    t = torch.randn((nfield, NLAT, NLON), device='cuda', dtype=torch.float32)
    cm = torch.zeros((NLAT, NLON), device='cuda', dtype=torch.float32)
    cs = torch.ones((NLAT, NLON), device='cuda', dtype=torch.float32)
    base = min(p.data_ptr() for p in (x, t, cm, cs))
    rel = lambda p: (p.data_ptr() - base) // 4
    off_x = np.arange(nfield, dtype=np.int64) * slab + rel(x)
    off_t = np.arange(nfield, dtype=np.int64) * slab + rel(t)
    off_a = np.zeros(nfield, dtype=np.int64) + rel(cm)
    off_b = np.zeros(nfield, dtype=np.int64) + rel(cs)
    out = torch.zeros((nfield, 4, 1, 8), device='cuda', dtype=torch.float64)
    fn = lambda: ctx.ens_threshold_metrics(
        base, base, m, nfield * slab, off_x, off_t, 4, base, off_a, base,
        off_b, z, spec, False, out.data_ptr())
    ms = timeit(fn, args.steps)
    pts = nfield * slab
    report(f'ens_threshold_metrics M={m} 4 thresholds', ms,
           pts * (4 * m + 4), pts, 'grid_points',
           {'note': 'climatology mean/std slab (8 MB) is L2-resident'})
    del x
  f = torch.randn((nfield * 10, NLAT, NLON), device='cuda',
                  dtype=torch.float32)
  s = torch.rand((nfield * 10, NLAT, NLON), device='cuda',
                 dtype=torch.float32) + 0.5
  t = torch.randn((nfield * 10, NLAT, NLON), device='cuda',
                  dtype=torch.float32)
  nf = nfield * 10
  base = min(p.data_ptr() for p in (f, s, t, cm, cs))
  rel = lambda p: (p.data_ptr() - base) // 4
  offs = [np.arange(nf, dtype=np.int64) * slab + rel(p) for p in (f, s, t)]
  off_a = np.zeros(nf, dtype=np.int64) + rel(cm)
  off_b = np.zeros(nf, dtype=np.int64) + rel(cs)
  out = torch.zeros((nf, 4, 1, 8), device='cuda', dtype=torch.float64)
  for nq in (0, 4):
    fn = lambda: ctx.gaussian_metrics(
        base, base, base, offs[0], offs[1], offs[2], nq, base if nq else None,
        off_a if nq else None, base if nq else None, off_b if nq else None,
        z[:nq] if nq else None, spec, False, out.data_ptr())
    ms = timeit(fn, args.steps)
    cells = nf * slab
    report(f'gaussian_metrics nthreshold={nq}', ms, cells * 12, cells,
           'grid_cells')


def _card():
  """Card name and power limit of this run (a number depends on both)."""
  import subprocess
  import torch
  info = {'card': torch.cuda.get_device_name(0)}
  try:
    info['power_limit_W'] = float(subprocess.run(
        ['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits',
         '-i', '0'], capture_output=True, text=True, timeout=30,
        check=True).stdout.split()[0])
  except Exception:  # pylint: disable=broad-except
    info['power_limit_W'] = None
  return info


def climatology_bytes(nsel, ncell, nhour, nday, nstat, esize=4):
  """Bytes the climatology needs: every selected time step of every cell read
  once, every output written once.  The per-day moments stay in shared memory
  (20 B per day slot and cell), so they add no HBM traffic."""
  return nsel * ncell * esize + nstat * nhour * nday * ncell * 4


def bench_climatology(args):
  """Hourly explicit mean + std (scripts/compute_climatology.py's default
  method) on a device-resident 721 x 1440 series (4 years 6-hourly, 24 GB)
  and on a 13-level 121 x 240 series (5 years 6-hourly) streamed from host
  memory."""
  import time
  import numpy as np
  torch, _lib, ctx = setup()
  from weatherbench2_b200 import utils
  card = _card()
  hours = [0, 6, 12, 18]
  # device-resident
  times = np.arange(np.datetime64('2017-01-01', 'ns'),
                    np.datetime64('2021-01-01', 'ns'), np.timedelta64(6, 'h'))
  ncell = NLAT * NLON
  x = torch.empty((times.size, ncell), device='cuda', dtype=torch.float32)
  for i in range(0, times.size, 512):
    x[i:i + 512].normal_()
  plan, labels = utils._plan(times, slice('2017', '2020'), hours,  # pylint: disable=protected-access
                             utils.EXPLICIT, False, 61)
  mean = torch.empty((len(hours), labels.size, ncell), device='cuda')
  std = torch.empty_like(mean)
  fn = lambda: ctx.climatology(x.data_ptr(), _lib.F32, times.size, ncell, plan,
                               mean.data_ptr(), std.data_ptr())
  ms = timeit(fn, args.steps, warmup=1)
  nbytes = climatology_bytes(times.size, ncell, len(hours), labels.size, 2)
  report('climatology device 721x1440 6-hourly 4y hourly explicit mean+std',
         ms, nbytes, times.size * ncell, 'values', dict(
             card, input_GB=times.size * ncell * 4 / 1e9))
  del x, mean, std
  torch.cuda.empty_cache()
  # streamed from host memory
  times = np.arange(np.datetime64('2016-01-01', 'ns'),
                    np.datetime64('2021-01-01', 'ns'), np.timedelta64(6, 'h'))
  ncell = 13 * 121 * 240
  rs = np.random.default_rng(0)
  block = rs.standard_normal((61, ncell), dtype=np.float32)
  xh = np.empty((times.size, ncell), np.float32)
  for i in range(0, times.size, 61):
    xh[i:i + 61] = block[:times.size - i]
  plan, labels = utils._plan(times, slice('2016', '2020'), hours,  # pylint: disable=protected-access
                             utils.EXPLICIT, False, 61)
  mh = np.empty((len(hours), labels.size, ncell), np.float32)
  sh = np.empty_like(mh)
  run = lambda: ctx.climatology_host(xh.ctypes.data, _lib.F32, times.size,
                                     ncell, plan, utils.STREAM_BUDGET_BYTES,
                                     mh.ctypes.data, sh.ctypes.data)
  run()
  t0 = time.perf_counter()
  for _ in range(args.steps):
    run()
  s = (time.perf_counter() - t0) / args.steps
  # the pageable host -> device rate of this machine, 1 GiB
  probe = xh.reshape(-1)[:1 << 28]
  dev = torch.empty(probe.size, device='cuda', dtype=torch.float32)
  dev.copy_(torch.from_numpy(probe))
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  for _ in range(3):
    dev.copy_(torch.from_numpy(probe))
  torch.cuda.synchronize()
  h2d = 3 * probe.nbytes / (time.perf_counter() - t0) / 1e9
  nbytes = climatology_bytes(times.size, ncell, len(hours), labels.size, 2)
  gbs = nbytes / s / 1e9
  print(json.dumps(dict(
      card, kernel='climatology streamed 13x121x240 6-hourly 5y hourly '
      'explicit mean+std', ms=s * 1e3, algorithmic_GB=nbytes / 1e9,
      achieved_GBps=gbs, h2d_pageable_GBps=h2d, frac_of_h2d=gbs / h2d)),
        flush=True)


def bench_climatology_quantile(args):
  """Hourly explicit quantiles (0.1, 0.25, 0.5, 0.75, 0.9) and the SEEPS pair
  of a 121 x 240 field, 6-hourly 1990-2019 (5.1 GB), window 61: on the device
  and streamed from host memory.  Bytes: every selected step read once, every
  output written once.  Work: the sorted-window entries each output day's
  prefix pass scans, nyear * (window - 2) per (hour, day, cell)."""
  import time
  import numpy as np
  torch, _lib, ctx = setup()
  from weatherbench2_b200 import utils
  card = _card()
  hours, qs, window = [0, 6, 12, 18], [0.1, 0.25, 0.5, 0.75, 0.9], 61
  times = np.arange(np.datetime64('1990-01-01', 'ns'),
                    np.datetime64('2020-01-01', 'ns'), np.timedelta64(6, 'h'))
  ncell = 121 * 240
  plan, labels = utils._plan(times, slice('1990', '2019'), hours,  # pylint: disable=protected-access
                             utils.EXPLICIT, False, window)
  entries = len(hours) * labels.size * ncell * plan.nitem * (window - 2)
  x = torch.empty((times.size, ncell), device='cuda', dtype=torch.float32)
  gen = torch.Generator(device='cuda').manual_seed(0)
  for i in range(0, times.size, 4096):
    x[i:i + 4096].normal_(generator=gen)
  out = torch.empty((len(hours), len(qs), labels.size, ncell), device='cuda')
  fn = lambda: ctx.climatology_quantile(x.data_ptr(), _lib.F32, times.size,
                                        ncell, plan, qs, None, out.data_ptr(),
                                        None)
  ms = timeit(fn, args.steps, warmup=1)
  nbytes = climatology_bytes(times.size, ncell, len(hours), labels.size,
                             len(qs))
  report('climatology_quantile device 121x240 6-hourly 30y hourly window 61 '
         '5 quantiles', ms, nbytes, entries, 'window_entries',
         dict(card, input_GB=times.size * ncell * 4 / 1e9))
  # SEEPS on a precipitation-like field: about 40 % zeros
  wet = torch.empty_like(x)
  for i in range(0, times.size, 4096):
    wet[i:i + 4096].uniform_(generator=gen)
  x.abs_().mul_(1e-3).mul_((wet >= 0.4).float())
  del wet
  dry = torch.empty((len(hours), labels.size, ncell), device='cuda')
  fn = lambda: ctx.climatology_quantile(x.data_ptr(), _lib.F32, times.size,
                                        ncell, plan, [2 / 3], 0.25e-3,
                                        out.data_ptr(), dry.data_ptr())
  ms = timeit(fn, args.steps, warmup=1)
  nbytes = climatology_bytes(times.size, ncell, len(hours), labels.size, 2)
  report('climatology_quantile device 121x240 6-hourly 30y hourly window 61 '
         'SEEPS (40% zeros)', ms, nbytes, entries, 'window_entries',
         dict(card, note='window_entries counts every sample; dry ones '
              'never enter the window'))
  # the first workload from host memory
  del x, out, dry
  block = np.random.default_rng(1).standard_normal((4096, ncell),
                                                    dtype=np.float32)
  xh = np.empty((times.size, ncell), np.float32)
  for i in range(0, times.size, 4096):
    xh[i:i + 4096] = block[:times.size - i]
  torch.cuda.empty_cache()
  oh = np.empty((len(hours), len(qs), labels.size, ncell), np.float32)
  run = lambda: ctx.climatology_quantile_host(
      xh.ctypes.data, _lib.F32, times.size, ncell, plan, qs, None,
      utils.STREAM_BUDGET_BYTES, oh.ctypes.data, None)
  run()
  t0 = time.perf_counter()
  for _ in range(args.steps):
    run()
  s = (time.perf_counter() - t0) / args.steps
  nbytes = climatology_bytes(times.size, ncell, len(hours), labels.size,
                             len(qs))
  print(json.dumps(dict(
      card, kernel='climatology_quantile streamed 121x240 6-hourly 30y hourly '
      'window 61 5 quantiles', ms=s * 1e3, algorithmic_GB=nbytes / 1e9,
      achieved_GBps=nbytes / s / 1e9, window_entries_per_s=entries / s)),
        flush=True)


def resample_bytes(nouter, ntime, ninner, nout, nstat, esize=4, window=0,
                   block=256):
  """Bytes a time resample / rolling window needs: the input read once (plus,
  rolling, the w-1 halo rows each block of `block` outputs stages again) and
  every output written once."""
  halo = (window - 1) * -(-ntime // block) if window else 0
  return (nouter * (ntime + halo) * ninner + nstat * nouter * nout * ninner
          ) * esize


def bench_resample(args):
  """Device-resident 721 x 1440, 6-hourly for 2 years (12.1 GB): daily mean +
  min + max (resample 1D) and a rolling 7-day mean (28 steps); then a
  13 x 121 x 240 series, 6-hourly for 5 years, streamed from host memory:
  weekly mean."""
  import time
  import numpy as np
  import pandas as pd
  torch, _lib, ctx = setup()
  from weatherbench2_b200 import resampling
  card = _card()
  times = np.arange(np.datetime64('2019-01-01', 'ns'),
                    np.datetime64('2021-01-01', 'ns'), np.timedelta64(6, 'h'))
  ncell = NLAT * NLON
  x = torch.empty((times.size, ncell), device='cuda', dtype=torch.float32)
  gen = torch.Generator(device='cuda').manual_seed(0)
  for i in range(0, times.size, 512):
    x[i:i + 512].normal_(generator=gen)
  _, start, count = resampling._bins(times, pd.Timedelta('1D'), 'left')  # pylint: disable=protected-access
  out = [torch.empty((count.size, ncell), device='cuda') for _ in range(3)]
  fn = lambda: ctx.time_window_stats(
      x.data_ptr(), _lib.F32, 1, times.size, ncell, start, count, 0, False,
      out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr(), None)
  ms = timeit(fn, args.steps, warmup=2)
  nbytes = resample_bytes(1, times.size, ncell, count.size, 3)
  report('resample device 721x1440 6-hourly 2y daily mean+min+max', ms,
         nbytes, times.size * ncell, 'values',
         dict(card, input_GB=times.size * ncell * 4 / 1e9))
  del out
  roll = torch.empty_like(x)
  fn = lambda: ctx.time_window_stats(
      x.data_ptr(), _lib.F32, 1, times.size, ncell, None, None, 28, False,
      roll.data_ptr(), None, None, None)
  ms = timeit(fn, args.steps, warmup=2)
  nbytes = resample_bytes(1, times.size, ncell, times.size, 1, window=28)
  report('resample device 721x1440 6-hourly 2y rolling 7-day mean (w=28)', ms,
         nbytes, times.size * ncell, 'values', dict(card))
  del x, roll
  torch.cuda.empty_cache()
  # streamed from host memory: (time, level, lat, lon), weekly mean
  times = np.arange(np.datetime64('2016-01-01', 'ns'),
                    np.datetime64('2021-01-01', 'ns'), np.timedelta64(6, 'h'))
  ncell = 13 * 121 * 240
  block = np.random.default_rng(0).standard_normal((61, ncell),
                                                   dtype=np.float32)
  xh = np.empty((times.size, ncell), np.float32)
  for i in range(0, times.size, 61):
    xh[i:i + 61] = block[:times.size - i]
  _, start, count = resampling._bins(times, pd.Timedelta('7D'), 'left')  # pylint: disable=protected-access
  mh = np.empty((count.size, ncell), np.float32)
  run = lambda: ctx.time_window_stats_host(
      xh.ctypes.data, _lib.F32, 1, times.size, ncell, start, count, 0, False,
      resampling.STREAM_BUDGET_BYTES, mh.ctypes.data, None, None, None)
  run()
  t0 = time.perf_counter()
  for _ in range(args.steps):
    run()
  s = (time.perf_counter() - t0) / args.steps
  probe = xh.reshape(-1)[:1 << 28]  # the pageable host -> device rate, 1 GiB
  dev = torch.empty(probe.size, device='cuda', dtype=torch.float32)
  dev.copy_(torch.from_numpy(probe))
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  for _ in range(3):
    dev.copy_(torch.from_numpy(probe))
  torch.cuda.synchronize()
  h2d = 3 * probe.nbytes / (time.perf_counter() - t0) / 1e9
  nbytes = resample_bytes(1, times.size, ncell, count.size, 1)
  gbs = nbytes / s / 1e9
  print(json.dumps(dict(
      card, kernel='resample streamed 13x121x240 6-hourly 5y weekly mean',
      ms=s * 1e3, algorithmic_GB=nbytes / 1e9, achieved_GBps=gbs,
      h2d_pageable_GBps=h2d, frac_of_h2d=gbs / h2d)), flush=True)


def bench_wind_dynamics(args):
  """Device-resident 0.25-degree (time=4, level=13, 721, 1440) u, v, z:
  divergence (8 B read + 4 B written per cell), geostrophic wind speed (4 + 4),
  ageostrophic wind speed (12 + 4) and vertical velocity (8 + 4), next to a
  device copy (4 + 4) of the same field measured in the same run."""
  torch, _lib, ctx = setup()
  from weatherbench2_b200 import _derived_wind as dw
  card = _card()
  nouter, nlev = 4, 13
  lat = np.linspace(-90, 90, NLAT)
  lon = np.arange(NLON) * 0.25
  lat_tab, lat_uni = dw.gradient_table(lat)
  lon_tab, lon_uni = dw.gradient_table(lon)
  cos = np.cos(np.deg2rad(lat))
  cor = dw.coriolis_parameter(lat)
  pres = 100.0 * np.array([50, 100, 150, 200, 250, 300, 400, 500, 600, 700,
                           850, 925, 1000])
  shape = (nouter, nlev, NLAT, NLON)
  gen = torch.Generator(device='cuda').manual_seed(0)
  u = torch.empty(shape, device='cuda').normal_(0, 10, generator=gen)
  v = torch.empty(shape, device='cuda').normal_(0, 10, generator=gen)
  z = torch.empty(shape, device='cuda').normal_(5e4, 300, generator=gen)
  out = torch.empty(shape, device='cuda')
  ncell = u.numel()
  cases = [('divergence', dw.DIVERGENCE, 8),
           ('geostrophic_wind_speed', dw.GEOSTROPHIC_WIND_SPEED, 4),
           ('ageostrophic_wind_speed', dw.AGEOSTROPHIC_WIND_SPEED, 12),
           ('vertical_velocity', dw.VERTICAL_VELOCITY, 8)]
  for name, kind, read in cases:
    fn = lambda kind=kind: ctx.wind_dynamics(
        kind, u.data_ptr(), v.data_ptr(), z.data_ptr(), nouter, nlev, NLAT,
        NLON, NLON, 1, lat_tab, lat_uni, lon_tab, lon_uni, cos, cor, pres,
        out.data_ptr())
    ms = timeit(fn, args.steps)
    report(f'wind_dynamics {name} 4x13x721x1440', ms, ncell * (read + 4),
           ncell, 'cells', dict(card))
  ms = timeit(lambda: out.copy_(u), args.steps)
  report('device copy 4x13x721x1440 (torch copy_)', ms, ncell * 8, ncell,
         'cells', dict(card))


def bench_column_integral(args):
  """Device-resident 0.25-degree (time=4, level=37, 721, 1440) float32 q, u, v:
  integrated vapor transport over 300-1000 hPa (20 of the 37 levels: 3 x 4 B
  read per selected level and cell, 4 B written per cell) and eddy kinetic
  energy over all 37 levels (2 x 4 B read per level and cell, 4 B written) in
  both layouts, next to a device copy of q measured in the same run; all of it
  twice."""
  torch, _lib, ctx = setup()
  from weatherbench2_b200 import _derived_column as dc
  card = _card()
  level = np.array([1, 2, 3, 5, 7, 10, 20, 30, 50, 70, 100, 125, 150, 175,
                    200, 225, 250, 300, 350, 400, 450, 500, 550, 600, 650,
                    700, 750, 775, 800, 825, 850, 875, 900, 925, 950, 975,
                    1000])
  nouter, nlev, ncell = 4, level.size, NLAT * NLON
  shape = (nouter, nlev, NLAT, NLON)
  gen = torch.Generator(device='cuda').manual_seed(0)
  q = torch.empty(shape, device='cuda').uniform_(0, 0.02, generator=gen)
  u = torch.empty(shape, device='cuda').normal_(5, 12, generator=gen)
  v = torch.empty(shape, device='cuda').normal_(0, 8, generator=gen)
  out = torch.empty((nouter, NLAT, NLON), device='cuda')
  lev0 = int(np.searchsorted(level, 300))
  nsel = nlev - lev0
  off = lev0 * ncell * 4
  w_ivt = dc.level_weights(level[lev0:])
  w_all = dc.level_weights(level)
  cases = [
      ('IVT 300-1000 hPa (20 levels)', nsel * 12 + 4,
       lambda: ctx.column_integral(
           dc.IVT, _lib.F32, q.data_ptr() + off, u.data_ptr() + off,
           v.data_ptr() + off, nouter, nlev * ncell, nsel, ncell, 0, 0, w_ivt,
           out.data_ptr())),
      ('EKE (latitude, longitude)', nlev * 8 + 4,
       lambda: ctx.column_integral(
           dc.EKE, _lib.F32, None, u.data_ptr(), v.data_ptr(), nouter,
           nlev * ncell, nlev, ncell, NLON, 1, w_all, out.data_ptr())),
      ('EKE (longitude, latitude)', nlev * 8 + 4,
       lambda: ctx.column_integral(
           dc.EKE, _lib.F32, None, u.data_ptr(), v.data_ptr(), nouter,
           nlev * ncell, nlev, ncell, NLON, NLAT, w_all, out.data_ptr())),
  ]
  copy = torch.empty_like(q)
  for run in (1, 2):  # twice in one process, to show the spread
    for name, per_cell, fn in cases:
      ms = timeit(fn, args.steps)
      report(f'column_integral {name} 4x37x721x1440', ms,
             nouter * ncell * per_cell, nouter * ncell, 'columns',
             dict(card, run=run))
    ms = timeit(lambda: copy.copy_(q), args.steps)
    report('device copy 4x37x721x1440 (torch copy_)', ms, q.numel() * 8,
           q.numel(), 'cells', dict(card, run=run))


def bench_thermo(args):
  """Device-resident 0.25-degree (time=4, level=37, 721, 1440) float32 data:
  the lapse rate (T and Z read, the float32 result written: 12 B per cell) and
  the relative humidity on int64 levels (T and q read, the float64 result
  written: 16 B per cell), in the (latitude, longitude) and (longitude,
  latitude) layouts and with the level axis innermost, next to a device copy
  measured in the same run; all of it twice."""
  torch, _lib, ctx = setup()
  from weatherbench2_b200 import _derived_wind as dw
  card = _card()
  level = np.array([1, 2, 3, 5, 7, 10, 20, 30, 50, 70, 100, 125, 150, 175,
                    200, 225, 250, 300, 350, 400, 450, 500, 550, 600, 650,
                    700, 750, 775, 800, 825, 850, 875, 900, 925, 950, 975,
                    1000])
  nouter, nlev, ncell = 4, level.size, NLAT * NLON
  coef, uniform = dw.gradient_table(level)
  pressure = level.astype(np.float64)
  gen = torch.Generator(device='cuda').manual_seed(0)
  n = nouter * nlev * ncell
  t = torch.empty(n, device='cuda').normal_(250, 20, generator=gen)
  z = torch.empty(n, device='cuda').normal_(5e4, 3e4, generator=gen)
  q = torch.empty(n, device='cuda').uniform_(0, 0.02, generator=gen)
  out = torch.empty(n, device='cuda')
  out64 = torch.empty(n, device='cuda', dtype=torch.float64)
  # (nouter, nlev, ninner) of each layout: both spatial layouts give the
  # entries the same sizes; level innermost makes every column contiguous
  layouts = [('(latitude, longitude)', nouter, nlev, ncell),
             ('(longitude, latitude)', nouter, nlev, ncell),
             ('level innermost', nouter * ncell, nlev, 1)]
  copy = torch.empty_like(t)
  for run in (1, 2):  # twice in one process, to show the spread
    for name, no, nl, ni in layouts:
      ms = timeit(lambda no=no, nl=nl, ni=ni: ctx.lapse_rate(
          _lib.F32, t.data_ptr(), z.data_ptr(), no, nl, ni, coef, uniform,
          out.data_ptr()), args.steps)
      report(f'lapse_rate {name} 4x37x721x1440', ms, n * 12, n, 'cells',
             dict(card, run=run))
      ms = timeit(lambda no=no, nl=nl, ni=ni: ctx.relative_humidity(
          _lib.F32, _lib.F64, t.data_ptr(), q.data_ptr(), no, nl, ni,
          pressure, out64.data_ptr()), args.steps)
      report(f'relative_humidity float32 -> float64 {name} 4x37x721x1440', ms,
             n * 16, n, 'cells', dict(card, run=run))
    ms = timeit(lambda: copy.copy_(t), args.steps)
    report('device copy 4x37x721x1440 (torch copy_)', ms, n * 8, n, 'cells',
           dict(card, run=run))


def precip_bytes(nouter, ntime, ninner, window, esize=4, block=256):
  """Bytes a precipitation accumulation needs: the input read once plus the
  `window` halo rows each block of `block` outputs stages again, and the
  output written once."""
  halo = window * -(-ntime // block)
  return (nouter * (ntime + halo) * ninner + nouter * ntime * ninner) * esize


def bench_precip_accumulation(args):
  """Device-resident 721 x 1440 cumulative precipitation: 2 inits x 41
  six-hourly leads with w = 4 (24 h), 1 init x 241 hourly leads with w = 24;
  then 2 x 41 x 181 x 360 streamed from host memory; each next to a torch
  device copy of the same bytes measured in the same run."""
  import time
  torch, _lib, ctx = setup()
  card = _card()
  ncell = NLAT * NLON
  gen = torch.Generator(device='cuda').manual_seed(0)
  for nouter, ntime, window in ((2, 41, 4), (1, 241, 24)):
    x = torch.empty((nouter, ntime, ncell), device='cuda').exponential_(
        1e3, generator=gen).cumsum(1)
    out = torch.empty_like(x)
    fn = lambda: ctx.precip_accumulation(  # noqa: E731
        x.data_ptr(), _lib.F32, nouter, ntime, ncell, window, True,
        out.data_ptr())
    ms = timeit(fn, args.steps)
    report(f'precip_accumulation device {nouter}x{ntime}x721x1440 w={window}',
           ms, precip_bytes(nouter, ntime, ncell, window), x.numel(),
           'values', dict(card))
    ms = timeit(lambda: out.copy_(x), args.steps)
    report(f'device copy {nouter}x{ntime}x721x1440 (torch copy_)', ms,
           2 * x.numel() * 4, x.numel(), 'values', dict(card))
    del x, out
  torch.cuda.empty_cache()
  from weatherbench2_b200 import resampling
  ncell = 181 * 360
  rs = np.random.default_rng(0)
  xh = np.cumsum(rs.exponential(1e-3, size=(2, 41, ncell)).astype(np.float32),
                 axis=1, dtype=np.float32)
  oh = np.empty_like(xh)
  run = lambda: ctx.precip_accumulation_host(  # noqa: E731
      xh.ctypes.data, _lib.F32, 2, 41, ncell, 4, True,
      resampling.STREAM_BUDGET_BYTES, oh.ctypes.data)
  run()
  t0 = time.perf_counter()
  for _ in range(args.steps):
    run()
  s = (time.perf_counter() - t0) / args.steps
  dev = torch.empty(xh.size, device='cuda')
  src = torch.from_numpy(xh.reshape(-1))
  dev.copy_(src)
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  for _ in range(args.steps):
    dev.copy_(src)
    src.copy_(dev)
  torch.cuda.synchronize()
  rt = (time.perf_counter() - t0) / args.steps
  print(json.dumps(dict(
      card, kernel='precip_accumulation streamed 2x41x181x360 w=4',
      ms=s * 1e3, algorithmic_GB=precip_bytes(2, 41, ncell, 4) / 1e9,
      torch_pageable_roundtrip_ms=rt * 1e3)), flush=True)


def _torch_sort_quantile(torch, x, q):
  """What a user would write without the kernel: torch.sort along the sample
  dim, then a gather of the order statistics and numpy's lerp (no NaN)."""
  n = x.shape[1]
  v = [(n - 1) * float(k) for k in q]
  i = [min(int(np.floor(t)), n - 1) for t in v]
  j = [min(k + 1, n - 1) for k in i]
  g = torch.tensor([t - k for t, k in zip(v, i)], device=x.device,
                   dtype=torch.float64).view(1, -1, 1)
  s = torch.sort(x, dim=1).values
  a = s.index_select(1, torch.tensor(i, device=x.device)).double()
  b = s.index_select(1, torch.tensor(j, device=x.device)).double()
  return a + (b - a) * g


def bench_quantile(args):
  """wb2_quantile on device-resident float32 series against torch.sort plus a
  gather in the same run: an ensemble (n = 50), one year of 6-hourly steps
  (n = 1460, also with 1 and 20 quantiles), 30 years at 1.5 degrees
  (n = 43,828), the longitude axis (ninner = 1); then a 13-level year streamed
  from host NumPy.  Bytes: the input once plus the float64 output once."""
  import time
  torch, _lib, ctx = setup()
  card = _card()
  q5 = [0.01, 0.1, 0.5, 0.9, 0.99]
  ncell = NLAT * NLON
  cases = [('ensemble 4x50x721x1440', (4, 50, ncell), q5),
           ('one year 1460x721x1440', (1, 1460, ncell), q5),
           ('one year 1460x721x1440 nq=1', (1, 1460, ncell), [0.5]),
           ('one year 1460x721x1440 nq=20', (1, 1460, ncell),
            list(np.linspace(0.025, 0.975, 20))),
           ('1990-2019 43828x121x240', (1, 43828, 121 * 240), q5),
           ('longitude (1460x721)x1440x1', (1460 * 721, 1440, 1), q5)]
  gen = torch.Generator(device='cuda').manual_seed(0)
  for name, (nouter, n, ninner), q in cases:
    x = torch.empty((nouter, n, ninner), device='cuda').normal_(
        1e5, 1.0, generator=gen)
    out = torch.empty((len(q), nouter, ninner), device='cuda',
                      dtype=torch.float64)
    fn = lambda: ctx.quantile(x.data_ptr(), _lib.F32, nouter, n, ninner,  # noqa: E731
                              q, False, out.data_ptr())
    nbytes = x.numel() * 4 + out.numel() * 8
    ms = timeit(fn, args.steps)
    report(f'quantile device {name} nq={len(q)}', ms, nbytes,
           nouter * ninner, 'cells', dict(card, nsample=n))
    if 'nq=' not in name:
      ref = _torch_sort_quantile(torch, x, q)
      got = out.permute(1, 0, 2)
      assert torch.equal(torch.isnan(got), torch.isnan(ref)), name
      del ref, got
      torch.cuda.empty_cache()
      try:
        ms = timeit(lambda: _torch_sort_quantile(torch, x, q),  # noqa: E731
                    max(1, args.steps // 2), warmup=1)
        report(f'torch.sort + gather {name} nq={len(q)}', ms, nbytes,
               nouter * ninner, 'cells', dict(card, nsample=n))
      except torch.cuda.OutOfMemoryError:
        print(json.dumps(dict(card, kernel=f'torch.sort + gather {name}',
                              ms=None, error='out of memory')), flush=True)
    del x, out
    torch.cuda.empty_cache()
  from weatherbench2_b200 import preprocessing
  n, ninner = 1460, 13 * 121 * 240
  xh = torch.empty((1, n, ninner), device='cuda').normal_(
      280.0, 10.0, generator=gen).cpu().numpy()
  oh = np.empty((len(q5), 1, ninner))
  run = lambda: ctx.quantile_host(  # noqa: E731
      xh.ctypes.data, _lib.F32, 1, n, ninner, q5, False,
      preprocessing.QUANTILE_STREAM_BUDGET_BYTES, oh.ctypes.data)
  run()
  t0 = time.perf_counter()
  for _ in range(args.steps):
    run()
  s = (time.perf_counter() - t0) / args.steps
  dev = torch.empty(xh.size, device='cuda')
  src = torch.from_numpy(xh.reshape(-1))
  dev.copy_(src)
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  for _ in range(args.steps):
    dev.copy_(src)
  torch.cuda.synchronize()
  h2d = (time.perf_counter() - t0) / args.steps
  print(json.dumps(dict(
      card, kernel='quantile streamed host 1460x13x121x240 nq=5',
      ms=s * 1e3, algorithmic_GB=(xh.nbytes + oh.nbytes) / 1e9,
      torch_pageable_h2d_ms=h2d * 1e3)), flush=True)


def bench_average(args):
  """wb2_average against (x * w).nansum / count in torch, per statistic, in the
  same run: a global latitude-weighted mean of 1464 steps at 721 x 1440 (K R),
  (time, longitude) means of 124 steps x 13 levels (R K R), a time-mean map
  (R K), all three raw moments over (longitude, latitude), one cell over the
  whole array; then 1464 steps x 13 x 121 x 240 streamed from host NumPy, next
  to the pageable host-to-device rate.  Bytes: the input once plus the
  outputs once; the share is of the data sheet's 3.35 TB/s unless a measured
  peak is given."""
  import time
  torch, _lib, ctx = setup()
  from weatherbench2_b200 import _spatial as sp
  card = _card()
  gen = torch.Generator(device='cuda').manual_seed(0)
  ncell = NLAT * NLON
  w_lat = sp.lat_weights(np.linspace(-90, 90, NLAT))

  def field(shape):
    x = torch.empty(shape, device='cuda', dtype=torch.float32)
    flat = x.view(-1)
    for i in range(0, flat.numel(), 1 << 28):
      flat[i:i + (1 << 28)].normal_(280.0, 10.0, generator=gen)
    flat[::1000003] = float('nan')
    return x

  def run(name, x, shape, stats, base, weights=None, wdiv=1):
    k0, _, k1, _, k2 = shape
    dt = torch.float64 if weights is not None else torch.float32
    outs = {s: torch.empty(k0 * k1 * k2, device='cuda',
                           dtype=torch.float64 if s == 'frac' else dt)
            for s in stats}
    fn = lambda: ctx.average(x.data_ptr(), _lib.F32, shape, True,  # noqa: E731
                             **{s: o.data_ptr() for s, o in outs.items()},
                             weights=weights, wdiv=wdiv)
    nbytes = x.numel() * 4 + sum(o.numel() * o.element_size()
                                 for o in outs.values())
    ms = timeit(fn, args.steps, warmup=1)
    report(f'average device {name}', ms, nbytes, x.numel(), 'samples',
           dict(card, shape=list(shape), stats=list(stats)))
    ref = base()
    for s, r in zip(stats, ref):
      torch.testing.assert_close(outs[s].double(), r.reshape(-1).double(),
                                 rtol=1e-5, atol=1e-6, equal_nan=True)
    del ref
    torch.cuda.empty_cache()
    ms = timeit(base, max(1, args.steps // 2), warmup=1)
    report(f'torch nansum / count {name}', ms, nbytes, x.numel(), 'samples',
           card)

  # global latitude-weighted mean per step: [1464][721 * 1440]
  x = field((1464, NLAT, NLON))
  wt = torch.from_numpy(w_lat).cuda()[:, None]

  def base_global():
    cnt = (~x.isnan()).sum((1, 2))
    return [(x * wt).nansum((1, 2)) / cnt]
  run('global lat-weighted mean 1464x721x1440 (K R)', x,
      (1464, ncell, 1, 1, 1), ('mean',), base_global, w_lat, NLON)
  del x
  torch.cuda.empty_cache()
  # [124 time][13 level][721][1440]
  x = field((124, 13, NLAT, NLON))

  def base_tlon():
    return [x.nansum((0, 3)) / (~x.isnan()).sum((0, 3))]
  run('(time, longitude) 124x13x721x1440 (R K R)', x,
      (1, 124, 13 * NLAT, NLON, 1), ('mean',), base_tlon)

  def base_tmap():
    return [x.nansum(0) / (~x.isnan()).sum(0)]
  run('time-mean map 124x13x721x1440 (R K)', x, (1, 124, 1, 1, 13 * ncell),
      ('mean',), base_tmap)

  def base_moments():
    cnt = (~x.isnan()).sum((2, 3))
    return [x.nansum((2, 3)) / cnt, (x * x).nansum((2, 3)) / cnt,
            cnt.double() / ncell]
  run('three moments 124x13x721x1440 (K R)', x, (124 * 13, ncell, 1, 1, 1),
      ('mean', 'mean_sq', 'frac'), base_moments)

  def base_all():
    return [x.nansum() / (~x.isnan()).sum()]
  run('reduce-all 124x13x721x1440 (one cell)', x, (1, x.numel(), 1, 1, 1),
      ('mean',), base_all)
  del x
  torch.cuda.empty_cache()
  # streamed from host NumPy: (time, longitude) of [1464][13][121][240]
  from weatherbench2_b200 import preprocessing
  shape = (1, 1464, 13 * 121, 240, 1)
  xh = field((1464, 13, 121, 240)).cpu().numpy()
  oh = np.empty(13 * 121, np.float32)
  runh = lambda: ctx.average_host(  # noqa: E731
      xh.ctypes.data, _lib.F32, shape, True,
      preprocessing.AVERAGE_STREAM_BUDGET_BYTES, mean=oh.ctypes.data)
  runh()
  t0 = time.perf_counter()
  for _ in range(args.steps):
    runh()
  s = (time.perf_counter() - t0) / args.steps
  dev = torch.empty(xh.size, device='cuda')
  src = torch.from_numpy(xh.reshape(-1))
  dev.copy_(src)
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  for _ in range(args.steps):
    dev.copy_(src)
  torch.cuda.synchronize()
  h2d = xh.nbytes / ((time.perf_counter() - t0) / args.steps) / 1e9
  gbs = xh.nbytes / s / 1e9
  print(json.dumps(dict(
      card, kernel='average streamed host (time, longitude) 1464x13x121x240',
      ms=s * 1e3, algorithmic_GB=xh.nbytes / 1e9, achieved_GBps=gbs,
      h2d_pageable_GBps=h2d, frac_of_h2d=gbs / h2d)), flush=True)


def bench_slab_gather(args):
  """wb2_slab_gather (the copy of weatherbench2_b200.reindexing) against the
  same gather in torch (index_select, masked_fill with NaN, .to(float32)),
  on both of its kernels: probabilistic forecasts (10 members x 61 leads x 28
  inits) from 4 years of 6-hourly 13x121x240 truth and a 0.25-degree 13-level
  forecast on valid time (slabs of 377,520 and 13.5 M elements: the chunked
  16-byte kernel), and 64x32 single-level forecasts (slabs of 2048: the flat
  kernel).  Bytes are the output written plus, per output slab, its source
  slab read.  Then a memmap truth through the host entry: bytes moved and rate."""
  import tempfile
  import time
  import pandas as pd
  torch, _lib, ctx = setup()
  from weatherbench2_b200 import reindexing as ri
  card = _card()
  rng = np.random.default_rng(0)

  def prob_offsets(ntime_truth, members, leads, inits):
    truth = pd.date_range('1990-01-01', periods=ntime_truth, freq='6h')
    out_t = pd.date_range('1992-01-01', periods=inits, freq='6h')
    sampled = ri.get_sampled_init_times(
        out_t, climatology_start_year=1990, climatology_end_year=1992,
        ensemble_size=members, seed=1)
    deltas = np.arange(leads) * np.timedelta64(6, 'h')
    need = sampled[:, None, :] + deltas[None, :, None]
    return truth.get_indexer(need.reshape(-1)).astype(np.int64)

  def run_case(name, src, pos, slab, out_dtype):
    """pos: source slab per output slab, -1 for NaN."""
    to = torch.float32 if out_dtype == _lib.F32 else torch.float64
    out = torch.empty((pos.size, slab), dtype=to, device='cuda')
    code = _lib.F32 if src.dtype == torch.float32 else _lib.F64
    offsets = np.where(pos < 0, -1, pos * slab)
    dev = lambda: ctx.slab_gather(src.data_ptr(), code, src.numel(), slab,
                                  pos.size, offsets, out.data_ptr(), out_dtype)
    src2 = src.view(-1, slab)
    idx = torch.from_numpy(np.maximum(pos, 0)).cuda()
    miss = torch.from_numpy(pos < 0).cuda()[:, None]
    base = lambda: src2.index_select(0, idx).masked_fill_(miss, float('nan')).to(to)
    dev()
    ref = base()
    torch.cuda.synchronize()
    for r in range(0, pos.size, 256):  # equal, NaN where NaN (in row blocks)
      a, b = out[r:r + 256], ref[r:r + 256]
      assert torch.equal(a.isnan(), b.isnan()) and torch.equal(
          torch.nan_to_num(a), torch.nan_to_num(b)), name
    del ref, a, b
    # every output slab written once and its source slab read once (a
    # source slab used by several outputs is read again unless L2 holds it)
    nread = int((pos >= 0).sum()) * slab * src.element_size()
    nbytes = out.numel() * out.element_size() + nread
    for label, fn in (('wb2_slab_gather', dev), ('torch baseline', base)):
      ms = timeit(fn, args.steps)
      report(f'slab_gather {name} [{label}]', ms, nbytes, pos.size, 'slabs',
             card)
    del out
    torch.cuda.empty_cache()

  ncell = 13 * 121 * 240
  ntruth = 4 * 1461
  truth = torch.empty((ntruth, ncell), dtype=torch.float32, device='cuda')
  truth.normal_()
  run_case('prob 10x61x28 from 4y 6-hourly 13x121x240 f32', truth,
           prob_offsets(ntruth, 10, 61, 28), ncell, _lib.F32)
  del truth
  torch.cuda.empty_cache()
  # forecast on valid time: 8 inits 12 h apart, 5 leads 6 h apart, valid_and_delta
  init = np.arange(8) * 12
  leads = np.arange(5) * 6
  kept = np.arange(0, 5, 2)
  times = np.unique(init[:, None] + leads[kept][None, :])
  ii = pd.Index(init).get_indexer((times[:, None] - leads[kept][None, :]).reshape(-1))
  pos = np.where(ii < 0, -1, ii * 5 + np.tile(kept, times.size))
  slab = 13 * NLAT * NLON
  for dt, tag in ((torch.float32, 'f32'), (torch.float64, 'f64')):
    fc = torch.empty((8 * 5, slab), dtype=dt, device='cuda')
    fc.normal_()
    run_case(f'valid time 13x721x1440 {tag}->f32 ({pos.size} slabs)', fc, pos,
             slab, _lib.F32)
    del fc
    torch.cuda.empty_cache()
  small = torch.empty((ntruth, 64 * 32), dtype=torch.float32, device='cuda')
  small.normal_()
  run_case('prob 10x61x280 from 4y 6-hourly 64x32 f32 (flat kernel)', small,
           prob_offsets(ntruth, 10, 61, 280), 64 * 32, _lib.F32)
  del small
  torch.cuda.empty_cache()

  # host entry: one year of 13x121x240 truth on a memmap, 10 x 61 x 4 slabs
  with tempfile.TemporaryDirectory() as tmp:
    nt = 1464
    mm = np.memmap(os.path.join(tmp, 'truth.f32'), np.float32, 'w+',
                   shape=(nt, ncell))
    block = rng.standard_normal((61, ncell), dtype=np.float32)
    for i in range(0, nt, 61):
      mm[i:i + 61] = block[:nt - i]
    mm.flush()
    pos = prob_offsets(ntruth, 10, 61, 4) % nt
    offsets = np.where(pos < 0, -1, pos * ncell)
    out = ctx.pinned_result((pos.size, ncell), np.float32)
    run = lambda: ctx.slab_gather_host(
        mm.ctypes.data, _lib.F32, mm.size, ncell, pos.size, offsets,
        ri.STREAM_BUDGET_BYTES, out.ctypes.data, _lib.F32)
    run()
    ctx.reset_transfer_stats()
    t0 = time.perf_counter()
    for _ in range(args.steps):
      run()
    s = (time.perf_counter() - t0) / args.steps
    st = ctx.transfer_stats()
    moved = (st['h2d_bytes'] + st['d2h_bytes']) / args.steps
    probe = np.asarray(mm[:256]).reshape(-1)
    dev = torch.empty(probe.size, device='cuda', dtype=torch.float32)
    dev.copy_(torch.from_numpy(probe))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(3):
      dev.copy_(torch.from_numpy(probe))
    torch.cuda.synchronize()
    h2d = 3 * probe.nbytes / (time.perf_counter() - t0) / 1e9
    print(json.dumps(dict(
        card, kernel='slab_gather host memmap 1y 13x121x240 -> 10x61x4 slabs',
        ms=s * 1e3, h2d_GB=st['h2d_bytes'] / args.steps / 1e9,
        d2h_GB=st['d2h_bytes'] / args.steps / 1e9,
        moved_GBps=moved / s / 1e9, h2d_pageable_GBps=h2d)), flush=True)
    del mm


if __name__ == '__main__':
  ap = argparse.ArgumentParser()
  ap.add_argument('--kernel', required=True,
                  choices=['ens', 'energy', 'det', 'regrid', 'spectrum',
                           'maps', 'threshold', 'climatology',
                           'climatology_quantile', 'resample',
                           'wind_dynamics', 'precip_accumulation',
                           'column_integral', 'thermo', 'quantile',
                           'average', 'slab_gather'])
  ap.add_argument('--steps', type=int, default=10)
  ap.add_argument('--fields', type=int, default=39)
  ap.add_argument('--members', type=int, nargs='+', default=[50])
  a = ap.parse_args()
  {'ens': bench_ens, 'energy': bench_energy, 'det': bench_det, 'regrid': bench_regrid,
   'spectrum': bench_spectrum, 'maps': bench_maps,
   'threshold': bench_threshold,
   'climatology': bench_climatology,
   'climatology_quantile': bench_climatology_quantile,
   'resample': bench_resample,
   'wind_dynamics': bench_wind_dynamics,
   'precip_accumulation': bench_precip_accumulation,
   'column_integral': bench_column_integral,
   'thermo': bench_thermo,
   'quantile': bench_quantile,
   'average': bench_average,
   'slab_gather': bench_slab_gather}[a.kernel](a)

"""Time wb2_regrid_bilinear at 1440x721 -> 240x121 (0.25 deg -> 1.5 deg, both
with poles) over 222 fields, host clock around each call and a device synchronise, and print one JSON line.

  python benchmarks/bench_regrid_bilinear.py [--iters N] [--lib PATH]

--lib loads another build of libwb2b200.so, so two versions can be compared
by running the script once per library, alternating.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--iters', type=int, default=50)
  ap.add_argument('--warmup', type=int, default=5)
  ap.add_argument('--nfield', type=int, default=222)
  ap.add_argument('--lib', default=None)
  args = ap.parse_args()
  import torch
  from weatherbench2_b200 import _lib, regridding
  if args.lib:
    _lib.LIB_PATH = os.path.abspath(args.lib)
  src = regridding.Grid(longitudes=np.linspace(0, 360, 1440, endpoint=False),
                        latitudes=np.linspace(-90, 90, 721), periodic=True,
                        includes_poles=True)
  tgt = regridding.Grid(longitudes=np.linspace(0, 360, 240, endpoint=False),
                        latitudes=np.linspace(-90, 90, 121), periodic=True,
                        includes_poles=True)
  r = regridding.BilinearRegridder(src, tgt)
  ctx = _lib.default_context(0)
  x = torch.randn(args.nfield, 1440, 721, device='cuda') * 100 + 5e4
  y = torch.empty(args.nfield, 240, 121, device='cuda')
  for _ in range(args.warmup):
    r.regrid_device(ctx, x.data_ptr(), y.data_ptr(), args.nfield)
  ctx.synchronize()
  times = []
  for _ in range(args.iters):  # one call each: tap upload, launch, completion
    t0 = time.perf_counter()
    r.regrid_device(ctx, x.data_ptr(), y.data_ptr(), args.nfield)
    ctx.synchronize()
    times.append((time.perf_counter() - t0) * 1e3)
  prop = torch.cuda.get_device_properties(0)
  print(json.dumps({
      'op': 'regrid_bilinear', 'shape': '1440x721->240x121',
      'nfield': args.nfield, 'lib': args.lib or _lib.LIB_PATH,
      'median_ms': float(np.median(times)), 'min_ms': float(np.min(times)),
      'gpu': prop.name}))


if __name__ == '__main__':
  main()

"""TEST INFRASTRUCTURE: NumPy interpretation of wb2_average / wb2_average_host
(include/wb2b200.h) on top of `fake_ctx.FakeContext`, so that
preprocessing.compute_averages, moment_reduce and compute_statistical_moments
run end to end on a CPU.  It applies the entries' argument checks and
tests/average_oracle.py to the canonical [k0][r0][k1][r1][k2] array the
operators hand to the library (the kernels themselves are checked by the GPU
tests)."""
import math

import numpy as np

import average_oracle as ao
import fake_ctx
from fake_ctx import _view
from weatherbench2_b200 import _lib


class AverageFakeContext(fake_ctx.FakeContext):
  """FakeContext plus the average entries."""

  def average(self, x, dtype, shape, skipna, mean=0, mean_sq=0, frac=0,
              weights=None, wdiv=1, wlen=None):
    self.calls.append(('average', tuple(int(s) for s in shape), bool(skipna),
                       weights is not None, int(wdiv)))
    self._run(x, dtype, shape, skipna, mean, mean_sq, frac, weights, wdiv,
              wlen)

  def average_host(self, x, dtype, shape, skipna, budget, mean=0, mean_sq=0,
                   frac=0, weights=None, wdiv=1, wlen=None):
    self.calls.append(('average_host', tuple(int(s) for s in shape),
                       bool(skipna), weights is not None, int(wdiv),
                       int(budget)))
    self._run(x, dtype, shape, skipna, mean, mean_sq, frac, weights, wdiv,
              wlen)

  @staticmethod
  def _run(x, dtype, shape, skipna, mean, mean_sq, frac, weights, wdiv, wlen):
    k0, r0, k1, r1, k2 = (int(s) for s in shape)
    if dtype not in (_lib.F32, _lib.F64):
      raise _lib.Wb2Error(f'wb2_average: dtype must be WB2_F32 or WB2_F64 '
                          f'(got {dtype})')
    if r0 < 1 or r1 < 1:
      raise _lib.Wb2Error('wb2_average: reduced extents r0 and r1 must be '
                          '>= 1')
    if min(k0, k1, k2) < 0:
      raise _lib.Wb2Error('wb2_average: kept extents k0, k1 and k2 must be '
                          '>= 0')
    n = r0 * r1
    if weights is not None:
      wlen = len(weights) if wlen is None else wlen
      if wdiv < 1 or wlen < 1 or n % wdiv or (n // wdiv) % wlen:
        raise _lib.Wb2Error(f'wb2_average: weights (wdiv {wdiv}, wlen '
                            f'{wlen}) do not fit the sample index')
    if not (mean or mean_sq or frac):
      raise _lib.Wb2Error('wb2_average: no output requested: mean, mean_sq '
                          'and frac are NULL')
    ncell = k0 * k1 * k2
    if not ncell:
      return
    dt = np.float32 if dtype == _lib.F32 else np.float64
    x5 = _view(x, ncell * n, dt).reshape(k0, r0, k1, r1, k2)
    res = ao.canonical(x5, bool(skipna), None if weights is None else
                       np.asarray(weights, np.float64)[:wlen], wdiv)
    for ptr, a in zip((mean, mean_sq, frac), res):
      if ptr:
        _view(ptr, math.prod(a.shape), a.dtype)[...] = a.reshape(-1)


def installed():
  """Makes `_lib.default_context()` return an AverageFakeContext."""
  return fake_ctx.installed(AverageFakeContext)

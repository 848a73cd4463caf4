"""TEST INFRASTRUCTURE: NumPy interpretation of wb2_quantile /
wb2_quantile_host (include/wb2b200.h) on top of `fake_ctx.FakeContext`, so that
preprocessing.compute_quantiles runs end to end on a CPU.  It applies the
entries' argument checks and tests/quantile_oracle.py to the
[outer][n][inner] series the operator hands to the library (the kernels'
staging, sorting networks and radix select are checked by the GPU tests)."""
import numpy as np

import fake_ctx
import quantile_oracle as qo
from fake_ctx import _view
from weatherbench2_b200 import _lib


class QuantileFakeContext(fake_ctx.FakeContext):
  """FakeContext plus the quantile entries."""

  def quantile(self, x, dtype, nouter, nsample, ninner, quantiles, skipna,
               out, nquantile=None):
    self.calls.append(('quantile', int(nouter), int(nsample), int(ninner),
                       len(quantiles), bool(skipna)))
    self._run(x, dtype, nouter, nsample, ninner, quantiles, skipna, out,
              nquantile)

  def quantile_host(self, x, dtype, nouter, nsample, ninner, quantiles,
                    skipna, budget, out, nquantile=None):
    self.calls.append(('quantile_host', int(nouter), int(nsample),
                       int(ninner), len(quantiles), bool(skipna), int(budget)))
    self._run(x, dtype, nouter, nsample, ninner, quantiles, skipna, out,
              nquantile)

  @staticmethod
  def _run(x, dtype, nouter, nsample, ninner, quantiles, skipna, out,
           nquantile):
    nq = len(quantiles) if nquantile is None else nquantile
    if dtype not in (_lib.F32, _lib.F64):
      raise _lib.Wb2Error(f'wb2_quantile: dtype must be WB2_F32 or WB2_F64 '
                          f'(got {dtype})')
    if nsample < 1:
      raise _lib.Wb2Error('wb2_quantile: nsample must be >= 1')
    if nouter < 0 or ninner < 0:
      raise _lib.Wb2Error('wb2_quantile: nouter and ninner must be >= 0')
    if not 1 <= nq <= _lib.MAX_QUANTILES:
      raise _lib.Wb2Error(f'wb2_quantile: nquantile must be in 1..128 '
                          f'(got {nq})')
    for k, q in enumerate(quantiles[:nq]):
      if not 0 <= q <= 1:
        raise _lib.Wb2Error(f'wb2_quantile: quantiles[{k}] = {q} is not in '
                            '[0, 1]')
    if not nouter * ninner:
      return
    dt = np.float32 if dtype == _lib.F32 else np.float64
    n = nouter * nsample * ninner
    series = _view(x, n, dt).reshape(nouter, nsample, ninner)
    res = qo.quantile(series, list(quantiles[:nq]), bool(skipna))
    _view(out, nq * nouter * ninner, np.float64)[...] = res.reshape(-1)


def installed():
  """Makes `_lib.default_context()` return a QuantileFakeContext."""
  return fake_ctx.installed(QuantileFakeContext)

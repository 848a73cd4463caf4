"""TEST INFRASTRUCTURE: NumPy interpretation of wb2_precip_accumulation /
wb2_precip_accumulation_host (include/wb2b200.h), plus the rolling entries of
fake_ctx_resample, on top of `fake_ctx.FakeContext`, so that the precipitation
derived variables run end to end on a CPU.  It applies the entry's argument
checks and tests/precip_oracle.py to the [outer][time][inner] series the
operators hand to the library (the kernel's staging and in-place differences
are checked by the GPU tests)."""
import numpy as np

import fake_ctx
import fake_ctx_resample
import precip_oracle as po
from fake_ctx import _view
from weatherbench2_b200 import _lib

MAX_WINDOW = 1024  # staged steps of the kernel


class PrecipFakeContext(fake_ctx_resample.ResampleFakeContext):
  """ResampleFakeContext plus the precipitation accumulation entries."""

  def precip_accumulation(self, x, dtype, nouter, ntime, ninner, window,
                          clamp_negative, out):
    self.calls.append(('precip_accumulation', int(nouter), int(ntime),
                       int(ninner), int(window), bool(clamp_negative)))
    self._accumulate(x, dtype, nouter, ntime, ninner, window, clamp_negative,
                     out)

  def precip_accumulation_host(self, x, dtype, nouter, ntime, ninner, window,
                               clamp_negative, budget, out):
    self.calls.append(('precip_accumulation_host', int(nouter), int(ntime),
                       int(ninner), int(window), bool(clamp_negative),
                       int(budget)))
    self._accumulate(x, dtype, nouter, ntime, ninner, window, clamp_negative,
                     out)

  @staticmethod
  def _accumulate(x, dtype, nouter, ntime, ninner, window, clamp, out):
    if dtype not in (_lib.F32, _lib.F64):
      raise _lib.Wb2Error(f'wb2_precip_accumulation: dtype {dtype}')
    if min(nouter, ntime, ninner) < 0 or window < 1:
      raise _lib.Wb2Error('wb2_precip_accumulation: bad sizes or window')
    if window > MAX_WINDOW and window < ntime:
      raise _lib.Wb2Error('wb2_precip_accumulation: window too wide')
    n = nouter * ntime * ninner
    if not n:
      return
    dt = np.float32 if dtype == _lib.F32 else np.float64
    series = _view(x, n, dt).reshape(nouter, ntime, ninner)
    res = po.accumulate(series, window, bool(clamp), axis=1)
    _view(out, n, dt)[...] = res.reshape(-1)


def installed():
  """Makes `_lib.default_context()` return a PrecipFakeContext."""
  return fake_ctx.installed(PrecipFakeContext)

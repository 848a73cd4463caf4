"""TEST INFRASTRUCTURE: NumPy interpretation of wb2_time_window_stats /
wb2_time_window_stats_host (include/wb2b200.h) on top of
`fake_ctx.FakeContext`, so that weatherbench2_b200.resampling runs end to end
on a CPU.  It reads the [outer][time][inner] series and the bin tables the
operators hand to the library and applies the float64 oracle bin by bin (the
kernels' staging, sliding sums and van Herk extrema are checked by the GPU
tests)."""
import numpy as np

import fake_ctx
import resample_oracle as ro
from fake_ctx import _view
from weatherbench2_b200 import _lib


class ResampleFakeContext(fake_ctx.FakeContext):
  """FakeContext plus the time window entries."""

  def time_window_stats(self, x, dtype, nouter, ntime, ninner, bin_start,
                        bin_count, window, skipna, mean, min, max, sum):  # pylint: disable=redefined-builtin
    self.calls.append(('time_window_stats', int(nouter), int(ntime),
                       int(ninner), int(window)))
    self._run(x, dtype, nouter, ntime, ninner, bin_start, bin_count, window,
              skipna, (mean, min, max, sum))

  def time_window_stats_host(self, x, dtype, nouter, ntime, ninner, bin_start,
                             bin_count, window, skipna, budget, mean, min,  # pylint: disable=redefined-builtin
                             max, sum):  # pylint: disable=redefined-builtin
    self.calls.append(('time_window_stats_host', int(nouter), int(ntime),
                       int(ninner), int(window), int(budget)))
    self._run(x, dtype, nouter, ntime, ninner, bin_start, bin_count, window,
              skipna, (mean, min, max, sum))

  @staticmethod
  def _run(x, dtype, nouter, ntime, ninner, bin_start, bin_count, window,
           skipna, ptrs):
    assert (bin_start is None) == (window > 0), 'exactly one of bins / window'
    dt = np.float32 if dtype == _lib.F32 else np.float64
    series = _view(x, nouter * ntime * ninner, dt).reshape(nouter, ntime,
                                                          ninner)
    stats = [s for s, p in zip(ro.STATISTICS, ptrs) if p]
    if window:
      res = ro.rolling(series, window, stats, axis=1)
    else:
      res = ro.resample(series, bin_start, bin_count, stats, skipna, axis=1)
    for s, p in zip(ro.STATISTICS, ptrs):
      if p:
        _view(p, res[s].size, dt)[...] = res[s].astype(dt).reshape(-1)


def installed():
  """Makes `_lib.default_context()` return a ResampleFakeContext."""
  return fake_ctx.installed(ResampleFakeContext)

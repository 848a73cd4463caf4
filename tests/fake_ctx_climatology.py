"""TEST INFRASTRUCTURE: NumPy interpretation of wb2_climatology /
wb2_climatology_host (include/wb2b200.h) on top of `fake_ctx.FakeContext`, so
that weatherbench2_b200.utils runs end to end on a CPU.  It reads the same
index tables the operators hand to the library and applies the header's
definitions tap by tap (the kernel's sliding sums and float64 shift are checked
by the GPU tests)."""
import numpy as np

import fake_ctx
from fake_ctx import _quiet, _view
from weatherbench2_b200 import _lib


class ClimatologyFakeContext(fake_ctx.FakeContext):
  """FakeContext plus the climatology entries."""

  def climatology(self, x, dtype, ntime, ncell, plan, mean, std):
    self.calls.append(('climatology', int(ncell), plan.method))
    self._climatology(x, dtype, ntime, ncell, plan, mean, std)

  def climatology_host(self, x, dtype, ntime, ncell, plan, budget, mean, std):
    self.calls.append(('climatology_host', int(ncell), plan.method,
                       int(budget)))
    self._climatology(x, dtype, ntime, ncell, plan, mean, std)

  @staticmethod
  def _climatology(x, dtype, ntime, ncell, plan, mean, std):
    dt = np.float32 if dtype == _lib.F32 else np.float64
    series = _view(x, ntime * ncell, dt).reshape(ntime, ncell).astype(
        np.float64)
    if plan.nres:  # daily resample: skip-NaN mean of consecutive slabs
      src = np.full((plan.nres, ncell), np.nan)
      for i in range(plan.nres):
        c = int(plan.res_count[i])
        if c:
          s = int(plan.res_start[i])
          with _quiet():
            src[i] = np.nanmean(series[s:s + c], axis=0)
    else:
      src = series
    half = plan.window_size // 2
    taps = np.arange(-half, half + 1)
    tri = (half - np.abs(taps)).astype(np.float64)
    w = tri / (tri.sum() / plan.window_size)  # create_window_weights
    res = np.full((2, plan.nhour, plan.nday_out, ncell), np.nan)
    for h in range(plan.nhour):
      n = int(plan.hour_nday[h])
      it = plan.items[h, :n]
      vals = np.where((it >= 0)[..., None], src[np.maximum(it, 0)], np.nan)
      if plan.method == 0:  # explicit: fill, weighted mean / std
        f = plan.fill[h]
        fv = np.where((f >= 0)[:, None], src[np.maximum(f, 0)], np.nan)
        vals = np.where(np.isnan(vals), fv[None], vals)
      else:  # fast: groupby mean / std of each slot
        with _quiet():
          vals = np.stack([np.nanmean(vals, axis=1), np.nanstd(vals, axis=1)])
      for d in range(n):
        idx = (d + taps) % n
        row = plan.out_row[h, d]
        if plan.method == 0:
          win = vals[idx]  # (tap, year, cell)
          ok = ~np.isnan(win)
          wb = w[:, None, None]
          sw = (wb * ok).sum(axis=(0, 1))
          with np.errstate(invalid='ignore', divide='ignore'):
            m = np.where(ok, wb * win, 0).sum(axis=(0, 1)) / sw
            v = np.where(ok, wb * (win - m) ** 2, 0).sum(axis=(0, 1)) / sw
          res[0, h, row] = np.where(sw > 0, m, np.nan)
          res[1, h, row] = np.where(sw > 0, np.sqrt(v), np.nan)
        else:
          for q in range(2):
            with _quiet():
              res[q, h, row] = np.nanmean(vals[q][idx] * w[:, None], axis=0)
    for q, ptr in enumerate((mean, std)):
      if ptr:
        _view(ptr, res[q].size, np.float32)[...] = res[q].astype(
            np.float32).reshape(-1)


def installed():
  """Makes `_lib.default_context()` return a ClimatologyFakeContext."""
  return fake_ctx.installed(ClimatologyFakeContext)

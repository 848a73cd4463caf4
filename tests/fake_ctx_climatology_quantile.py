"""TEST INFRASTRUCTURE: NumPy interpretation of wb2_climatology_quantile /
wb2_climatology_quantile_host (include/wb2b200.h) on top of
`fake_ctx_climatology.ClimatologyFakeContext`, so that the quantile and SEEPS
operators of weatherbench2_b200.utils run end to end on a CPU.  It reads the
index tables the operators hand to the library and applies the header's
definitions to every window at once, cells vectorised (the kernel's sliding
sorted window is checked by the GPU tests)."""
import numpy as np

import fake_ctx
import fake_ctx_climatology
from fake_ctx import _quiet, _view
from weatherbench2_b200 import _lib


def _weighted_quantiles(vals, w, qs):
  """[q][cell] weighted type-7 quantiles of vals [sample][cell] (NaN skipped)
  with sample weights w [sample]; zero weights and NaN get weight 0 and sort
  to no effect."""
  wt = np.where(np.isnan(vals), 0.0, w[:, None])
  order = np.argsort(vals, axis=0, kind='stable')
  v = np.take_along_axis(vals, order, 0)
  wt = np.take_along_axis(wt, order, 0)
  s1, s2 = wt.sum(0), (wt ** 2).sum(0)
  out = np.full((len(qs), vals.shape[1]), np.nan)
  with np.errstate(invalid='ignore', divide='ignore'):
    nw = s1 ** 2 / s2
    c = np.concatenate([np.zeros((1, vals.shape[1])), np.cumsum(wt, 0)]) / s1
    for i, q in enumerate(qs):
      h = np.clip((nw - 1) * q + 1, 1, nw)
      u = np.maximum((h - 1) / nw, np.minimum(h / nw, c))
      dv = np.diff(u * nw - h + 1, axis=0)
      out[i] = np.where(wt > 0, v * dv, 0.0).sum(0)
  return np.where(s1 > 0, out, np.nan)


class QuantileFakeContext(fake_ctx_climatology.ClimatologyFakeContext):
  """ClimatologyFakeContext plus the quantile / SEEPS entries."""

  def climatology_quantile(self, x, dtype, ntime, ncell, plan, quantiles,
                           seeps_threshold, out, dry_fraction):
    self.calls.append(('climatology_quantile', int(ncell)))
    self._quantile(x, dtype, ntime, ncell, plan, quantiles, seeps_threshold,
                   out, dry_fraction)

  def climatology_quantile_host(self, x, dtype, ntime, ncell, plan, quantiles,
                                seeps_threshold, budget, out, dry_fraction):
    self.calls.append(('climatology_quantile_host', int(ncell), int(budget)))
    self._quantile(x, dtype, ntime, ncell, plan, quantiles, seeps_threshold,
                   out, dry_fraction)

  @staticmethod
  def _quantile(x, dtype, ntime, ncell, plan, quantiles, seeps_threshold,
                out, dry_fraction):
    assert plan.method == 0
    dt = np.float32 if dtype == _lib.F32 else np.float64
    series = _view(x, ntime * ncell, dt).reshape(ntime, ncell)
    if plan.nres:  # daily resample in float32, like wb2_ens_mean
      src = np.full((plan.nres, ncell), np.nan, np.float32)
      for i in range(plan.nres):
        c = int(plan.res_count[i])
        if c:
          s = int(plan.res_start[i])
          with _quiet():
            src[i] = np.nanmean(series[s:s + c].astype(np.float64), axis=0)
    else:
      src = series
    qs = np.asarray(quantiles, np.float64)
    seeps = seeps_threshold is not None
    thr = src.dtype.type(seeps_threshold) if seeps else None
    half = plan.window_size // 2
    taps = np.arange(-half, half + 1)
    w = (half - np.abs(taps)).astype(np.float64)
    res = np.full((plan.nhour, qs.size, plan.nday_out, ncell), np.nan)
    dry = np.full((plan.nhour, plan.nday_out, ncell), np.nan)
    for h in range(plan.nhour):
      n = int(plan.hour_nday[h])
      it = plan.items[h, :n]
      real = (it >= 0).any(axis=0)  # the hour's stacked years
      vals = np.where((it >= 0)[..., None], src[np.maximum(it, 0)], np.nan)
      f = plan.fill[h]
      fv = np.where((f >= 0)[:, None], src[np.maximum(f, 0)], np.nan)
      vals = np.where(np.isnan(vals), fv[None], vals)[:, real]
      for d in range(n):
        win = vals[(d + taps) % n]  # (tap, year, cell)
        wts = np.repeat(w, win.shape[1])
        flat = win.reshape(-1, ncell)
        if seeps:
          is_dry = flat < thr
          dry[h, plan.out_row[h, d]] = is_dry.mean(0)
          flat = np.where(is_dry, np.nan, flat)
        res[h, :, plan.out_row[h, d]] = _weighted_quantiles(
            flat.astype(np.float64), wts, qs)
    _view(out, res.size, np.float32)[...] = res.astype(np.float32).ravel()
    if seeps:
      _view(dry_fraction, dry.size, np.float32)[...] = dry.astype(
          np.float32).ravel()


def installed():
  """Makes `_lib.default_context()` return a QuantileFakeContext."""
  return fake_ctx.installed(QuantileFakeContext)

"""NumPy oracle of wb2_average / wb2_average_host (include/wb2b200.h, DESIGN.md
section 8g).  It restates the header's recipe, summation order included:
samples in chunks of 65536, inside a chunk 32 classes (s mod 32) each summed in
increasing s from +0.0, the class sums added as a xor butterfly, the chunk
partials added in chunk order from +0.0.  Every addition is one numpy float64
addition, so the kernels must match it bit for bit."""
import math

import numpy as np

CHUNK = 65536


def ordered_sum(y):
  """The header's float64 sum of each row of y [cells][n]."""
  y = np.asarray(y, np.float64)
  cells, n = y.shape
  total = np.zeros(cells)
  with np.errstate(invalid='ignore', over='ignore'):
    for c0 in range(0, n, CHUNK):
      seg = y[:, c0:c0 + CHUNK]
      m = -(-seg.shape[1] // 32)
      pad = np.zeros((cells, m * 32))  # + 0.0 leaves a sum (never -0.0) as is
      pad[:, :seg.shape[1]] = seg
      pad = pad.reshape(cells, m, 32)
      a = np.zeros((cells, 32))
      for i in range(m):
        a = a + pad[:, i]
      for off in (16, 8, 4, 2, 1):
        a = a[:, :off] + a[:, off:2 * off]
      total = total + a[:, 0]
  return total


def cell_stats(t, skipna, w=None):
  """(S1, S2, N) of t [cells][n] (float32 or float64), `w` the float64
  weight of each sample (None: unweighted)."""
  t = np.asarray(t)
  with np.errstate(over='ignore', invalid='ignore'):
    sq = np.square(t).astype(np.float64)  # rounded in the data type
    y = t.astype(np.float64)
    if w is not None:
      y = y * w
      sq = sq * w
  nan = np.isnan(t)
  if skipna:
    y = np.where(nan, 0.0, y)
    sq = np.where(nan, 0.0, sq)
  return ordered_sum(y), ordered_sum(sq), (~nan).sum(axis=1).astype(np.float64)


def finish(s1, s2, cnt, n, skipna, dtype):
  """mean, mean_sq (in `dtype`) and frac from the sums."""
  div = cnt if skipna else np.float64(n)
  with np.errstate(invalid='ignore', divide='ignore'):
    return ((s1 / div).astype(dtype), (s2 / div).astype(dtype),
            cnt / np.float64(n))


def sample_weights(n, weights, wdiv):
  s = np.arange(n)
  return np.asarray(weights, np.float64)[(s // wdiv) % len(weights)]


def canonical(x5, skipna, weights=None, wdiv=1):
  """The entries' outputs for x5 [k0][r0][k1][r1][k2]: (mean, mean_sq, frac),
  each [k0][k1][k2]."""
  k0, r0, k1, r1, k2 = x5.shape
  n = r0 * r1
  t = x5.transpose(0, 2, 4, 1, 3).reshape(k0 * k1 * k2, n)
  w = None if weights is None else sample_weights(n, weights, wdiv)
  s1, s2, cnt = cell_stats(t, skipna, w)
  dt = np.float64 if weights is not None else x5.dtype
  return tuple(a.reshape(k0, k1, k2)
               for a in finish(s1, s2, cnt, n, skipna, dt))


def average(x, axes, skipna=False, weights=None, weight_axis=None):
  """(mean, mean_sq, frac) of x over `axes`, shaped like the kept axes in
  order.  Samples follow the reduced axes in input order (the operators'
  order both in place and after their transposed copy); `weights` is a
  vector along `weight_axis`."""
  axes = sorted(a % x.ndim for a in axes)
  keep = [a for a in range(x.ndim) if a not in axes]
  t = np.transpose(x, keep + axes)
  kshape = tuple(x.shape[a] for a in keep)
  n = math.prod(x.shape[a] for a in axes)
  t = t.reshape(math.prod(kshape), n)
  w = None
  if weights is not None:
    i = axes.index(weight_axis)
    wdiv = math.prod(x.shape[a] for a in axes[i + 1:])
    w = sample_weights(n, weights, wdiv)
  s1, s2, cnt = cell_stats(t, skipna, w)
  dt = np.float64 if weights is not None else x.dtype
  return tuple(a.reshape(kshape) for a in finish(s1, s2, cnt, n, skipna, dt))

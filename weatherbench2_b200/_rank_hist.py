"""RankHistogram -- same class as weatherbench2/metrics.py:1894-2042 -- on top of
K10 (csrc/rank_hist.cu).  Imported into `weatherbench2_b200.metrics`.
"""
from __future__ import annotations

import typing as t

import numpy as np

from weatherbench2_b200 import _ensemble as ens
from weatherbench2_b200 import _spatial as sp
from weatherbench2_b200 import metrics as m
from weatherbench2_b200 import xarray_lite as xl


class RankHistogram(ens.EnsembleMetric):
  """Histogram of truth's rank with respect to the ensemble members.

  `compute_chunk` gives the one-hot encoding of the rank with a trailing `bins`
  dimension (K + 1 bins, or `num_bins` dividing K + 1); averaging over time
  (`compute`, fused into the kernel) gives the histogram.  NaN values are
  treated as larger than any other; `skipna` is ignored (metrics.py:1911).

  Tie-breaking: the reference perturbs truth and members by uniform noise
  smaller than a quarter of the smallest gap (:1960-1987), which only reorders
  exact ties; the kernel places the truth uniformly among the members equal to
  it.  The draws come from a hash of `seed` (entropy from the OS when None),
  not from NumPy's PCG64 stream: without ties the result is identical to the
  reference, with ties it has the same distribution.
  """

  def __init__(self, ensemble_dim: str = ens.REALIZATION,
               num_bins: t.Optional[int] = None,
               break_ties_randomly: bool = True,
               seed: t.Optional[int] = None):
    super().__init__(ensemble_dim=ensemble_dim)
    self.num_bins = num_bins
    self._break_ties_randomly = break_ties_randomly
    self._seed = seed

  def __hash__(self):
    return id(self)

  def _num_bins_actual(self, ensemble_size: int) -> int:
    """metrics.py:1938-1946."""
    default_n_bins = ensemble_size + 1
    if self.num_bins is None:
      return default_n_bins
    if default_n_bins % self.num_bins:
      raise ValueError(
          f'Cannot bin data with {ensemble_size=} into {self.num_bins} bins')
    return self.num_bins

  def _hist(self, forecast, truth, reduce_dim):
    n_ensemble = ens._get_n_ensemble(forecast, self.ensemble_dim)  # pylint: disable=protected-access
    nbins = self._num_bins_actual(n_ensemble)
    seed = self._seed
    if seed is None:
      seed = int(np.random.SeedSequence().entropy) & (2**64 - 1)
    ctx = m._context()  # pylint: disable=protected-access
    names = m._common_vars(forecast, truth)  # pylint: disable=protected-access
    out = xl.Dataset()
    for name, f_da, t_da, x_op, t_op in m._paired_operands(  # pylint: disable=protected-access
        forecast, truth, np.float32):
      hist, dims = sp.run_rank_histogram(
          ctx, x_op, t_op, self.ensemble_dim, nbins, reduce_dim,
          self._break_ties_randomly, seed + names.index(name))
      coords = m._map_coords(dims, f_da, t_da)  # pylint: disable=protected-access
      coords.pop(self.ensemble_dim, None)
      coords['bins'] = xl.Coord(('bins',), np.arange(nbins))
      out[name] = xl.DataArray(hist, tuple(dims) + ('bins',), coords, name)
    return out

  def compute_chunk(self, forecast, truth, region=None, skipna=False):
    del region, skipna  # ignored, like the reference
    return self._hist(forecast, truth, None)

  def compute(self, forecast, truth, region=None, skipna=False):
    del region, skipna
    result = self._hist(forecast, truth, m._avg_dim(forecast))  # pylint: disable=protected-access
    return result.assign_attrs(ensemble_size=forecast.sizes[self.ensemble_dim])


@xl.boundary
def central_reliability(hist):
  """Reliability diagram for central histogram probabilities
  (weatherbench2/metrics.py:2045-2126), computed on an already reduced rank
  histogram (a handful of numbers per variable -- result assembly like the
  final `sum / weight_sum`, not kernel work).

  For N bins the probability that truth was less extreme than the central
  2(k+1) - N%2 bins, k = 0 .. N//2 - 1 + N%2, indexed by the probability a
  perfectly calibrated forecast would give, `desired_prob` (with the integer
  `prob_index` as a coordinate along it).
  """
  single = isinstance(hist, xl.DataArray)
  ds = xl.Dataset({hist.name or '_': hist}) if single else hist
  n_bins = ds.sizes['bins']
  if n_bins < 3:
    raise ValueError(f'Too few bins. {n_bins=} but should be >= 3')
  half, odd = n_bins // 2, n_bins % 2
  # label-based like the reference's .sel (bins are 0 .. N-1)
  bins = np.asarray(ds.coords['bins'].values) if 'bins' in ds.coords else (
      np.arange(n_bins))
  left_idx = xl.label_slice_indices(bins, slice(None, half - 1))
  right_idx = xl.label_slice_indices(bins, slice(half + odd, None))
  desired = np.ones(left_idx.size)
  if odd:
    desired = np.concatenate(([0.5], desired))
  desired = np.cumsum(desired)
  desired = desired / desired[-1]
  out = xl.Dataset(attrs=ds.attrs)
  for name in ds.keys():
    da = ds[name]
    if 'bins' not in da.dims:
      out[name] = da
      continue
    ax = da.dims.index('bins')
    h = np.moveaxis(np.asarray(da.values), ax, -1)
    # cumulative sum from the centre outwards: left half reversed + right half
    probs = np.cumsum(h[..., left_idx[::-1]] + h[..., right_idx], axis=-1)
    other = tuple(d for d in da.dims if d != 'bins')
    if odd:
      center = h[..., int(xl._lookup(bins, np.array([half]))[0])]  # pylint: disable=protected-access
      probs = np.concatenate([center[..., None], center[..., None] + probs],
                             axis=-1)
      # xr.concat puts the expanded prob_index dimension first
      data, dims = np.moveaxis(probs, -1, 0), ('desired_prob',) + other
    else:
      data = np.moveaxis(probs, -1, ax)
      dims = da.dims[:ax] + ('desired_prob',) + da.dims[ax + 1:]
    coords = {k: c for k, c in da.coords.items() if 'bins' not in c.dims}
    coords['desired_prob'] = xl.Coord(('desired_prob',), desired)
    coords['prob_index'] = xl.Coord(('desired_prob',), np.arange(desired.size))
    out[name] = xl.DataArray(data, dims, coords, name, da.attrs)
  return out[list(out.keys())[0]] if single else out

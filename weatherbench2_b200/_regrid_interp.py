"""Nearest-neighbour and bilinear regridders -- same classes as
weatherbench2/regridding.py:212-294 -- on top of K8 (csrc/regrid_interp.cu).

Imported into `weatherbench2_b200.regridding`; use them from there.  The host
part resolves what the reference does with a BallTree (nearest) or with
`jnp.interp`'s searchsorted / clamping / periodic wrap-around (bilinear) into
index / fraction tables; the kernels only gather and interpolate.
"""
from __future__ import annotations

import functools
from typing import Optional

import numpy as np

from weatherbench2_b200 import _lib
from weatherbench2_b200 import regridding as rg

_F32 = np.float32  # JAX default precision (x64 off) of the reference
_TAP = _F32(-1)    # fraction of a tap jnp.interp returns as it is


def nearest_neighbor_indices(source_grid: 'rg.Grid', target_grid: 'rg.Grid'
                             ) -> np.ndarray:
  """Haversine nearest-neighbour indices from source to target, the same
  BallTree query as regridding.py:212-228 (indices into the raveled
  (lon, lat) source slab)."""
  from sklearn.neighbors import BallTree  # pylint: disable=import-outside-toplevel

  def points(grid):
    # (lat, lon) in radians of every cell of the raveled (lon, lat) slab:
    # index = i_lon * nlat + i_lat, like the reference's meshgrid + ravel
    lat = np.deg2rad(np.asarray(grid.latitudes, dtype=np.float64))
    lon = np.deg2rad(np.asarray(grid.longitudes, dtype=np.float64))
    return np.column_stack([np.tile(lat, lon.size), np.repeat(lon, lat.size)])

  tree = BallTree(points(source_grid), metric='haversine')
  return tree.query(points(target_grid), k=1, return_distance=False)[:, 0]


def _jnp_remainder(x, period):
  """`x % period` as jnp.remainder computes it: C fmod, plus `period` where the
  nonzero remainder has the other sign (-0.0 stays -0.0, unlike np.mod)."""
  r = np.fmod(x, period)
  return np.where((r != 0) & ((r < 0) != (period < 0)), r + period,
                  r).astype(x.dtype)


def interp_taps(x, xp, clamp: bool, period: Optional[float] = None):
  """Taps of `jnp.interp(x, xp, fp, left, right, period)` in float32:
  (i0, i1, t) such that f = fp[i0] + t * (fp[i1] - fp[i0]).  i0 = -1 where the
  result is NaN (outside `xp` when `clamp` is False), with i1 = -1 too.  Where
  jnp.interp returns a tap value through `where` -- fp[0] / fp[-1] outside `xp`
  when `clamp` is True (jnp.interp's default left / right), fp[i-1] where
  |dx| <= spacing(eps) -- the taps are i1 = i0 and t = -1, and the kernel passes
  fp[i0] through untouched.  A genuine fraction is never negative, and
  `i0 == i1` alone does not mean a `where`: a one-longitude periodic axis has
  i0 == i1 == 0 and t = x / 360, and jnp.interp lerps there too.  Read as a
  plain lerp, fp + (-1) * (fp - fp) is still fp for every finite tap."""
  x = np.asarray(x, dtype=_F32)
  xp = np.asarray(xp, dtype=_F32)
  n = xp.size
  if period is not None:
    p = np.abs(_F32(period))
    x = _jnp_remainder(x, p)
    xp_m = _jnp_remainder(xp, p)
    order = np.argsort(xp_m, kind='stable')
    xp_s = xp_m[order]
    xp_ext = np.concatenate([xp_s[-1:] - p, xp_s, xp_s[:1] + p]).astype(_F32)
    src = np.concatenate([order[-1:], order, order[:1]])
  else:
    xp_ext, src = xp, np.arange(n)
  i = np.clip(np.searchsorted(xp_ext, x, side='right'), 1, xp_ext.size - 1)
  dx = (xp_ext[i] - xp_ext[i - 1]).astype(_F32)
  delta = (x - xp_ext[i - 1]).astype(_F32)
  eps = np.spacing(np.finfo(_F32).eps)
  dx0 = np.abs(dx) <= eps
  t = np.where(dx0, _TAP, delta / np.where(dx0, _F32(1), dx)).astype(_F32)
  i0 = src[i - 1].astype(np.int32)
  i1 = np.where(dx0, i0, src[i]).astype(np.int32)
  if period is None:
    lo, hi = x < xp[0], x > xp[-1]
    if clamp:
      i0 = np.where(lo, 0, np.where(hi, n - 1, i0)).astype(np.int32)
      i1 = np.where(lo | hi, i0, i1).astype(np.int32)
      t = np.where(lo | hi, _TAP, t).astype(_F32)
    else:
      i0 = np.where(lo | hi, -1, i0).astype(np.int32)
      i1 = np.where(lo | hi, -1, i1).astype(np.int32)
  return i0, i1, t


class NearestRegridder(rg.Regridder):
  """Regrid with nearest-neighbour interpolation (regridding.py:231-247)."""

  @functools.cached_property
  def indices(self):
    return nearest_neighbor_indices(self.source, self.target)

  def __hash__(self):
    return hash((self.source, self.target))

  def regrid_device(self, ctx: _lib.Context, src_ptr: int, dst_ptr: int,
                    nfield: int, src_stride: Optional[int] = None,
                    dst_stride: Optional[int] = None):
    ns = self.source.shape[0] * self.source.shape[1]
    nt = self.target.shape[0] * self.target.shape[1]
    ctx.regrid_gather(src_ptr, dst_ptr, nfield, src_stride or ns,
                      dst_stride or nt, ns, self.indices)


class BilinearRegridder(rg.Regridder):
  """Regrid with bilinear interpolation (regridding.py:256-294)."""

  @functools.cached_property
  def _taps(self):
    lat = interp_taps(self.target.latitudes, self.source.latitudes,
                      clamp=self.source.includes_poles)
    if self.source.periodic:
      lon = interp_taps(self.target.longitudes, self.source.longitudes,
                        clamp=True, period=360)
    else:
      lon = interp_taps(self.target.longitudes, self.source.longitudes,
                        clamp=False)
    return lon, lat

  def __hash__(self):
    return hash((self.source, self.target))

  def regrid_device(self, ctx: _lib.Context, src_ptr: int, dst_ptr: int,
                    nfield: int, src_stride: Optional[int] = None,
                    dst_stride: Optional[int] = None):
    ns = self.source.shape[0] * self.source.shape[1]
    nt = self.target.shape[0] * self.target.shape[1]
    lon, lat = self._taps
    ctx.regrid_bilinear(src_ptr, dst_ptr, nfield, src_stride or ns,
                        dst_stride or nt, self.source.shape, lon, lat)

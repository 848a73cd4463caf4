"""Conservative lat/lon regridding -- `Grid`, `Regridder` and
`ConservativeRegridder` with the API of weatherbench2/regridding.py:117-209,
297-536; the contraction runs in csrc/regrid.cu (banded stencil, one pass).

The weight matrices are built here with the reference's formulas (cell-overlap
areas along latitude, periodic interval overlaps along longitude) in float32,
the precision JAX uses by default, and handed to the kernel in CSR form.
Nearest / bilinear regridders (regridding.py:212-294): _regrid_interp.py.
NumPy inputs are streamed through double-buffered device staging
(wb2_regrid_conservative_host); CUDA tensors stay on the device.
"""
from __future__ import annotations

import dataclasses
import enum
import functools
from typing import Optional

import numpy as np

from weatherbench2_b200 import _lib
from weatherbench2_b200 import _streamed
from weatherbench2_b200 import xarray_lite as xl

_DT = np.float32


def _assert_increasing(x: np.ndarray) -> None:
  # regridding.py:297-299
  if not (np.diff(x) > 0).all():
    raise ValueError(f'array is not increasing: {x}')


class LongitudeScheme(enum.Enum):
  """Where a global longitude axis starts (regridding.py:43-48)."""
  START_AT_ZERO = enum.auto()   # 0, d, 2d, ..., 360 - d
  CENTER_AT_ZERO = enum.auto()  # -180 + d/2, ..., 180 - d/2


class LatitudeSpacing(enum.Enum):
  """Latitude node placement (regridding.py:51-54)."""
  EQUIANGULAR_WITH_POLES = enum.auto()
  EQUIANGULAR_WITHOUT_POLES = enum.auto()
  CUSTOM = enum.auto()  # e.g. Gaussian grids: nodes are given, not generated


def latitude_values(latitude_spacing: LatitudeSpacing, num: int) -> np.ndarray:
  """`num` equiangular latitudes, pole to pole or cell-centred
  (regridding.py:57-67)."""
  if latitude_spacing == LatitudeSpacing.EQUIANGULAR_WITH_POLES:
    edge = 90.0
  elif latitude_spacing == LatitudeSpacing.EQUIANGULAR_WITHOUT_POLES:
    edge = 90.0 - 90.0 / num  # half a cell inside the poles
  else:
    raise ValueError(f'Unhandled {latitude_spacing=}')
  return np.linspace(-edge, edge, num=num)


def longitude_values(longitude_scheme: LongitudeScheme, num: int) -> np.ndarray:
  """`num` equally spaced longitudes covering the circle once
  (regridding.py:70-82)."""
  step = 360 / num
  if longitude_scheme == LongitudeScheme.START_AT_ZERO:
    first = 0.0
  elif longitude_scheme == LongitudeScheme.CENTER_AT_ZERO:
    first = -180 + step / 2
  else:
    raise ValueError(f'Unhandled {longitude_scheme=}')
  return np.linspace(first, first + 360 - step, num=num)


def _check_global_coverage(longitudes: np.ndarray, latitudes: np.ndarray,
                           tolerance: float) -> None:
  """Raises unless the nodes span the globe to within `tolerance` degrees:
  latitude -90 .. 90 and longitude 0 .. 360 or -180 .. 180
  (regridding.py:88-114)."""
  lo_lat, hi_lat = float(np.min(latitudes)), float(np.max(latitudes))
  lo_lon, hi_lon = float(np.min(longitudes)), float(np.max(longitudes))

  def near(value, *targets):
    return any(abs(value - x) < tolerance for x in targets)

  if not near(lo_lat, -90):
    raise ValueError(
        f'min latitude must be within ±{tolerance} of -90, found {lo_lat}')
  if not near(hi_lat, 90):
    raise ValueError(
        f'max latitude must be within ±{tolerance} of 90, found {hi_lat}')
  if not near(lo_lon, 0, -180):
    raise ValueError(f'min longitude must be within ±{tolerance} of 0 or -180, '
                     f'found {lo_lon}')
  if not near(hi_lon, 360, 180):
    raise ValueError(f'max longitude must be within ±{tolerance} of 360 or '
                     f'+180, found {hi_lon}')


@dataclasses.dataclass(frozen=True)
class Grid:
  """Rectilinear grid (regridding.py:117-179)."""

  longitudes: np.ndarray = dataclasses.field(kw_only=True)
  latitudes: np.ndarray = dataclasses.field(kw_only=True)
  periodic: bool = dataclasses.field(kw_only=True)
  includes_poles: bool = dataclasses.field(kw_only=True)

  def __post_init__(self):
    _assert_increasing(np.asarray(self.latitudes))

  @classmethod
  def from_degrees(cls, lon: np.ndarray, lat: np.ndarray) -> 'Grid':
    """Legacy constructor (regridding.py:155-160)."""
    return cls(longitudes=lon, latitudes=lat, periodic=True,
               includes_poles=True)

  @property
  def shape(self) -> tuple[int, int]:
    return (len(self.longitudes), len(self.latitudes))

  def _to_tuple(self):
    return (tuple(np.asarray(self.longitudes).tolist()),
            tuple(np.asarray(self.latitudes).tolist()), self.periodic,
            self.includes_poles)

  def __eq__(self, other):
    return isinstance(other, Grid) and self._to_tuple() == other._to_tuple()

  def __hash__(self):
    return hash(self._to_tuple())


# ---- latitude weights (regridding.py:302-373) --------------------------------
def _latitude_cell_bounds(x, include_poles=True):
  if include_poles:
    initial = np.array([-90], dtype=x.dtype)
    final = np.array([90], dtype=x.dtype)
  else:
    initial = x[:1] - (x[1] - x[0]) / 2
    final = x[-1:] + (x[-1] - x[-2]) / 2
  return np.concatenate([initial, (x[:-1] + x[1:]) / 2, final])


def _latitude_area_from_bounds(lower, upper):
  return np.sin(np.deg2rad(upper)) - np.sin(np.deg2rad(lower))


def _conservative_latitude_weights(source_points, target_points,
                                   source_includes_poles,
                                   target_includes_poles) -> np.ndarray:
  """(target, source) matrix, rows sum to 1; NaN rows where the source grid
  does not cover the target cell (regridding.py:341-373)."""
  src = np.asarray(source_points, dtype=_DT)
  tgt = np.asarray(target_points, dtype=_DT)
  _assert_increasing(src)
  _assert_increasing(tgt)
  sb = _latitude_cell_bounds(src, source_includes_poles)
  tb = _latitude_cell_bounds(tgt, target_includes_poles)
  upper = np.minimum(tb[1:, None], sb[None, 1:])
  lower = np.maximum(tb[:-1, None], sb[None, :-1])
  overlap = (upper > lower) * _latitude_area_from_bounds(lower, upper)
  coverage = np.sum(overlap, axis=1, keepdims=True)
  with np.errstate(invalid='ignore', divide='ignore'):
    weights = overlap / coverage
  if not source_includes_poles:
    tbb = _latitude_cell_bounds(tgt, target_includes_poles)
    target_areas = _latitude_area_from_bounds(tbb[:-1], tbb[1:])[:, None]
    is_covered = np.isclose(coverage, target_areas, rtol=1e-3)
    weights = np.where(is_covered, weights, np.nan)
  return weights.astype(_DT)


# ---- longitude weights (regridding.py:376-499) -------------------------------
def _align_phase_with(x, target, period):
  if period is None:
    return x
  shift_down = x > target + period / 2
  shift_up = x < target - period / 2
  return x + period * shift_up - period * shift_down


def _periodic_upper_lower_bounds(x, period):
  if period is not None:
    x = x % period
    x_plus = _align_phase_with(np.roll(x, -1), x, period)
    x_minus = _align_phase_with(np.roll(x, +1), x, period)
  else:
    x_plus = np.concatenate([x[1:], x[-1:] + (x[-1] - x[-2])])
    x_minus = np.concatenate([x[:1] - (x[1] - x[0]), x[:-1]])
  return (x + x_plus) / 2, (x_minus + x) / 2


def _conservative_longitude_weights(source_points, target_points,
                                    source_periodic,
                                    target_periodic) -> np.ndarray:
  """(target, source) matrix (regridding.py:462-499)."""
  src = np.asarray(source_points, dtype=_DT)
  tgt = np.asarray(target_points, dtype=_DT)
  if len(tgt) < 3 and target_periodic:
    raise ValueError(
        'Need 3 or more target points else overlap is not well defined. Found'
        f' {len(tgt)}')
  _assert_increasing(src)
  _assert_increasing(tgt)
  t_up, t_lo = _periodic_upper_lower_bounds(tgt, 360 if target_periodic
                                            else None)
  s_up, s_lo = _periodic_upper_lower_bounds(src, 360 if source_periodic
                                            else None)
  x0, x1 = t_lo[:, None], t_up[:, None]
  y0 = _align_phase_with(s_lo[None, :], x0, 360)
  y1 = _align_phase_with(s_up[None, :], x0, 360)
  overlap = np.maximum(np.minimum(x1, y1) - np.maximum(x0, y0), 0)
  coverage = np.sum(overlap, axis=1, keepdims=True)
  with np.errstate(invalid='ignore', divide='ignore'):
    weights = overlap / coverage
  if not source_periodic:
    target_lengths = (t_up - t_lo)[:, None]
    is_covered = np.isclose(coverage, target_lengths, rtol=1e-3)
    weights = np.where(is_covered, weights, np.nan)
  return weights.astype(_DT)


@dataclasses.dataclass(frozen=True)
class Regridder:
  """Base class for regridding (regridding.py:182-209)."""

  source: Grid
  target: Grid

  def regrid_device(self, ctx: _lib.Context, src_ptr: int, dst_ptr: int,
                    nfield: int, src_stride: Optional[int] = None,
                    dst_stride: Optional[int] = None):
    """Raw device-pointer entry: `nfield` float32 slabs (lon, lat) -> slabs."""
    raise NotImplementedError

  def _fields(self, field) -> tuple[int, tuple]:
    """The field count and result shape of `field`, (..., lon, lat)."""
    shape = tuple(field.shape)
    if shape[-2:] != self.source.shape:
      raise ValueError(f'expected trailing dims {self.source.shape}, got '
                       f'{shape[-2:]}')
    batch = shape[:-2]
    return int(np.prod(batch)), batch + self.target.shape

  def regrid_array(self, field):
    """(..., lon, lat) -> (..., lon_target, lat_target), float32 like the
    reference (JAX default).  NumPy in -> NumPy out; CUDA tensor in -> out."""
    ctx = _lib.default_context()
    nfield, tshape = self._fields(field)
    return _streamed.run_whole(
        [field], [(tshape, np.float32)],
        lambda i, o: self.regrid_device(ctx, i[0], o[0], nfield),
        dtype=np.float32)[0]

  @xl.boundary
  def regrid_dataset(self, dataset):
    """Regrid a Dataset from source to target (regridding.py:193-209)."""
    lat = dataset['latitude'].values
    if not (np.diff(lat) > 0).all():
      dataset = dataset.isel(latitude=np.arange(lat.size)[::-1])
    assert (np.diff(dataset['latitude'].values) > 0).all()
    out = xl.Dataset(attrs=dataset.attrs)
    for name in dataset.keys():
      v = dataset[name]
      if 'longitude' not in v.dims or 'latitude' not in v.dims:
        out[name] = v
        continue
      dims = v.dims
      core_last = tuple(d for d in dims if d not in ('longitude', 'latitude')
                        ) + ('longitude', 'latitude')
      arr = self.regrid_array(v.transpose(*core_last).data)
      coords = {k: c for k, c in v.coords.items()
                if 'longitude' not in c.dims and 'latitude' not in c.dims}
      coords['longitude'] = xl.Coord(('longitude',),
                                     np.asarray(self.target.longitudes))
      coords['latitude'] = xl.Coord(('latitude',),
                                    np.asarray(self.target.latitudes))
      out[name] = xl.DataArray(arr, core_last, coords, name,
                               v.attrs).transpose(*dims)
    return out


class ConservativeRegridder(Regridder):
  """Linear conservative regridding, NaN-aware (regridding.py:502-536)."""

  @functools.cached_property
  def _weights(self):
    lon_w = _conservative_longitude_weights(
        self.source.longitudes, self.target.longitudes, self.source.periodic,
        self.target.periodic)
    lat_w = _conservative_latitude_weights(
        self.source.latitudes, self.target.latitudes,
        self.source.includes_poles, self.target.includes_poles)
    return _lib.CsrSpec(lon_w), _lib.CsrSpec(lat_w)

  def __hash__(self):
    return hash((self.source, self.target))

  def regrid_device(self, ctx: _lib.Context, src_ptr: int, dst_ptr: int,
                    nfield: int, src_stride: Optional[int] = None,
                    dst_stride: Optional[int] = None):
    """Raw device-pointer entry: `nfield` float32 slabs (lon, lat) -> slabs."""
    lon_w, lat_w = self._weights
    ns = self.source.shape[0] * self.source.shape[1]
    nt = self.target.shape[0] * self.target.shape[1]
    ctx.regrid_conservative(src_ptr, dst_ptr, nfield, src_stride or ns,
                            dst_stride or nt, lon_w, lat_w)

  def regrid_array(self, field):
    """As `Regridder.regrid_array`; NumPy input is streamed, so that the
    copies and kernels of neighbouring field groups overlap."""
    ctx = _lib.default_context()
    nfield, tshape = self._fields(field)
    ns = self.source.shape[0] * self.source.shape[1]
    nt = self.target.shape[0] * self.target.shape[1]
    return _streamed.place(
        field, [(tshape, np.float32)],
        lambda x, _, out: self.regrid_device(ctx, x.data_ptr(),
                                             out.data_ptr(), nfield),
        lambda x, _, out: ctx.regrid_conservative_host(
            x.ctypes.data, out.ctypes.data, nfield, ns, nt, *self._weights),
        dtype=np.float32)[0]


# Nearest / bilinear regridders live in _regrid_interp.py (they need Regridder).
from weatherbench2_b200._regrid_interp import (  # noqa: E402  pylint: disable=wrong-import-position
    BilinearRegridder, NearestRegridder, nearest_neighbor_indices)

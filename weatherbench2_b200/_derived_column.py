"""Column integrals over pressure level -- same classes as
weatherbench2/derived_variables.py:212-228 and 365-430: total column water,
integrated water transport and eddy kinetic energy, computed on the device
(csrc/column_integral.cu).  Imported into `weatherbench2_b200.derived_variables`.

A CUDA operand gives a CUDA tensor on its device, which the metric kernels
read in place; NumPy, memmap or lazily gathered input gives NumPy.  Float32
data gives float32, float64 gives float64.  The result has the input's dims
without `level`, in the same order, and the input's coords without those along
`level`, as xarray's integrate.
Numerics and deviations: include/wb2b200.h and DESIGN.md section 8h.
"""
from __future__ import annotations

import dataclasses
import typing as t

import numpy as np

from weatherbench2_b200 import _derived_wind
from weatherbench2_b200 import _lib
from weatherbench2_b200 import _streamed
from weatherbench2_b200 import derived_variables as dv
from weatherbench2_b200 import xarray_lite as xl

# `kind` of wb2_column_integral (include/wb2b200.h)
TOTAL_COLUMN, IVT, EKE = 0, 1, 2


def level_weights(level) -> np.ndarray:
  """w_k = 0.5 * (level[k+1] - level[k]) in float64: the `dx * 0.5` of
  xarray's trapz, for the levels actually integrated."""
  return np.diff(np.asarray(level, np.float64)) * 0.5


def column_integral(dataset, kind: int, names: t.Sequence[str],
                    level_slice: t.Optional[slice] = None):
  """One wb2_column_integral call on the named variables of `dataset` (q for
  TOTAL_COLUMN; q, u, v for IVT; u, v for EKE).  `level_slice` selects the
  levels as `.sel(level=level_slice)`: a contiguous run, passed to the kernel
  as a pointer offset and a count."""
  das = [dataset[n] for n in names]  # KeyError for a missing base variable
  ref = das[0]
  for name, da in zip(names, das):
    if 'level' not in da.dims:
      raise ValueError(f'{name!r} has no "level" dimension')
  if 'level' not in ref.coords:
    raise KeyError('level')
  _derived_wind.check_same_grid(names, das)
  # CUDA tensors stay where they are; anything else is read once as NumPy
  datas = [da.data if xl._is_torch(da.data) and da.data.is_cuda  # pylint: disable=protected-access
           else xl._np(da.data) for da in das]  # pylint: disable=protected-access
  dtypes = [str(x.dtype).replace('torch.', '') for x in datas]
  for name, dtype in zip(names, dtypes):
    if dtype not in ('float32', 'float64'):
      raise TypeError(f'variable {name!r} has dtype {dtype}: column integrals '
                      'take float32 or float64 data')
  dtype = np.result_type(*dtypes)
  level = np.asarray(ref.coords['level'].values)
  if level_slice is None:
    sel = np.arange(level.size)
  else:
    sel = xl.label_slice_indices(level, level_slice)  # KeyError: not monotonic
  lev0, nsel = (int(sel[0]), int(sel.size)) if sel.size else (0, 0)

  if kind == EKE:
    if 'longitude' not in ref.dims:
      raise ValueError(f'{names[0]!r} has no "longitude" dimension')
    spatial = tuple(d for d in ref.dims if d in ('latitude', 'longitude'))
  else:
    li = ref.dims.index('level')
    spatial = tuple(d for d in ref.dims[li + 1:])
  outer = tuple(d for d in ref.dims if d not in spatial + ('level',))
  work = outer + ('level',) + spatial
  perms = [None if da.dims == work else tuple(da.dims.index(d) for d in work)
           for da in das]
  shape = tuple(ref.sizes[d] for d in work)
  nouter = int(np.prod(shape[:len(outer)], dtype=np.int64))
  nlev = shape[len(outer)]
  ninner = int(np.prod(shape[len(outer) + 1:], dtype=np.int64))
  nlon = ref.sizes['longitude'] if kind == EKE else 0
  lon_stride = (1 if kind != EKE or spatial[-1] == 'longitude'
                else ninner // max(nlon, 1))
  weight = level_weights(level[sel]) if nsel > 1 else None
  out_shape = shape[:len(outer)] + shape[len(outer) + 1:]
  code = _lib.F64 if dtype == np.float64 else _lib.F32
  ctx = _lib.default_context()

  def call(ptrs, out):
    offset = lev0 * ninner * np.dtype(dtype).itemsize
    ptrs = [p + offset for p in ptrs]
    q, u, v = ((ptrs[0], None, None) if kind == TOTAL_COLUMN else
               (ptrs[0], ptrs[1], ptrs[2]) if kind == IVT else
               (None, ptrs[0], ptrs[1]))
    ctx.column_integral(kind, code, q, u, v, nouter, nlev * ninner, nsel,
                        ninner, nlon, lon_stride, weight, out[0])

  data, = _streamed.run_whole(datas, [(out_shape, dtype)], call, perms=perms,
                              dtype=dtype)
  out_dims = tuple(d for d in work if d != 'level')
  coords = {k: c for k, c in ref.coords.items() if 'level' not in c.dims}
  result = xl.DataArray(data, out_dims, coords)
  ref_dims = tuple(d for d in ref.dims if d != 'level')
  if out_dims != ref_dims:
    result = result.transpose(*ref_dims)
    if xl._is_torch(result.data):  # pylint: disable=protected-access
      result = xl.DataArray(result.data.contiguous(), ref_dims, coords)
  return result


@dataclasses.dataclass
class EddyKineticEnergy(_derived_wind._3DWindVariable):  # pylint: disable=protected-access
  """Eddy kinetic energy 0.5 * integral over level of u'^2 + v'^2, eddies
  being the deviation from the instantaneous zonal (NaN-skipping) mean
  (derived_variables.py:212-228).  Needs `level` and `longitude` dimensions
  and a `level` coordinate."""

  @property
  def core_dims(self):
    return (['level', 'longitude'], ['level', 'longitude']), ['longitude']

  def compute(self, dataset):
    return column_integral(dataset, EKE, [self.u_name, self.v_name])


@dataclasses.dataclass
class TotalColumnWater(dv.DerivedVariable):
  """Total column water (1 / 9.81) * integral of the species over level
  (derived_variables.py:365-385).

  Attributes:
    water_species_name: Name of water species to vertically integrate.
  """

  water_species_name: str = 'specific_humidity'

  @property
  def base_variables(self) -> list[str]:
    return [self.water_species_name]

  @property
  def core_dims(self):
    return (['level'],), []

  def compute(self, dataset):
    return column_integral(dataset, TOTAL_COLUMN, [self.water_species_name])


@dataclasses.dataclass
class IntegratedWaterTransport(dv.DerivedVariable):
  """Integrated horizontal water transport in a vertical column
  (derived_variables.py:388-430): (1 / 9.81) * sqrt(Iu^2 + Iv^2), Iu the
  integral over level of q * u on `.sel(level=slice(level_min, level_max))`.
  Integrated vapor transport (IVT) is a diagnostic for atmospheric rivers; the
  default levels are those of the GraphCast paper.  On descending levels that
  slice is empty, as in pandas, and the result is 0.

  Attributes:
    u_name: Name of wind U component.
    v_name: Name of wind V component.
    water_species_name: Name of water species to vertically integrate.
    level_min: Minimum pressure level to include.
    level_max: Maximum pressure level to include.
  """

  u_name: str = 'u_component_of_wind'
  v_name: str = 'v_component_of_wind'
  water_species_name: str = 'specific_humidity'
  level_min: t.Optional[float] = 300
  level_max: t.Optional[float] = 1000

  @property
  def base_variables(self) -> list[str]:
    return [self.u_name, self.v_name, self.water_species_name]

  @property
  def core_dims(self):
    return (['level'], ['level']), []

  def compute(self, dataset):
    return column_integral(
        dataset, IVT, [self.water_species_name, self.u_name, self.v_name],
        slice(self.level_min, self.level_max))

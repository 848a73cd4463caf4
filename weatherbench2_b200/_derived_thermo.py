"""Thermodynamic derived variables -- same classes as
weatherbench2/derived_variables.py:341-362 and 433-468: the lapse rate and the
relative humidity, computed on the device (csrc/thermo.cu).  Imported into
`weatherbench2_b200.derived_variables`.

A CUDA operand gives a CUDA tensor on its device, which the metric kernels
read in place; NumPy, memmap or lazily gathered input is read once as NumPy
and gives NumPy.  An operand in another dim order is permuted to the order of
the one whose dims the result takes: temperature's for the lapse rate,
specific humidity's for the relative humidity, as xarray's `dT_dp / dz_dp`
and `mixing_ratio / smr` order them.
Operands whose dims or sizes differ raise ValueError, where xarray would align
them.  Numerics and deviations: include/wb2b200.h and DESIGN.md section 8i.
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


def _operands(ds, names):
  """The named variables (KeyError for a missing one), each as a CUDA tensor
  or NumPy array, their permutations to the first one's dims (None for that
  order), and their common float dtype: integers are taken as float64, as
  np.gradient and NumPy's arithmetic take them."""
  das = [ds[n] for n in names]
  _derived_wind.check_same_grid(names, das)
  datas = [da.data if xl._is_torch(da.data) and da.data.is_cuda  # pylint: disable=protected-access
           else xl._np(da.data) for da in das]  # pylint: disable=protected-access
  dtypes = []
  for name, x in zip(names, datas):
    try:
      dtype = np.dtype(str(x.dtype).replace('torch.', ''))
    except TypeError:
      dtype = None
    if dtype is not None and dtype.kind in 'iu':
      dtype = np.dtype(np.float64)
    if dtype not in (np.float32, np.float64):
      raise TypeError(f'variable {name!r} has dtype {x.dtype}: the lapse rate '
                      'and relative humidity take float32, float64 or integer '
                      'data')
    dtypes.append(dtype)
  dims = das[0].dims
  perms = [None if da.dims == dims else tuple(da.dims.index(d) for d in dims)
           for da in das]
  return das, datas, perms, np.result_type(*dtypes)


def _split(shape, axis):
  """(nouter, n, ninner) of `shape` around `axis`."""
  nouter = int(np.prod(shape[:axis], dtype=np.int64))
  ninner = int(np.prod(shape[axis + 1:], dtype=np.int64))
  return nouter, shape[axis], ninner


def lapse_rate(dataset, temperature_name: str, geopotential_name: str):
  """One wb2_lapse_rate call: dT/dlevel / ((1 / 9.81) dZ/dlevel) with
  np.gradient's arithmetic along `level`, in temperature's dims."""
  names = [temperature_name, geopotential_name]
  das, datas, perms, dtype = _operands(dataset, names)
  temp = das[0]
  if 'level' not in temp.dims:
    raise ValueError(f'{temperature_name!r} has no "level" dimension')
  level = (temp.coords['level'] if 'level' in temp.coords
           else dataset.coords.get('level'))
  if level is None or tuple(level.dims) != ('level',):
    raise ValueError('Coordinate level does not exist.')
  coef, uniform = _derived_wind.gradient_table(level.values)  # ValueError: < 2
  dims = temp.dims
  shape = tuple(temp.sizes[d] for d in dims)
  nouter, nlev, ninner = _split(shape, dims.index('level'))
  code = _lib.F64 if dtype == np.float64 else _lib.F32
  ctx = _lib.default_context()

  def call(ptrs, out):
    ctx.lapse_rate(code, ptrs[0], ptrs[1], nouter, nlev, ninner, coef, uniform,
                   out[0])

  data, = _streamed.run_whole(datas, [(shape, dtype)], call,
                              perms=perms, dtype=dtype)
  coords = dict(das[1].coords)
  coords.update(temp.coords)
  return xl.DataArray(data, dims, coords)


def relative_humidity(dataset, temperature_name: str,
                      specific_humidity_name: str, pressure_name: str):
  """One wb2_relative_humidity call: MetPy's relative humidity from specific
  humidity with Bolton's saturation vapour pressure, T in K and the pressure
  coordinate in hPa, in specific humidity's dims."""
  names = [specific_humidity_name, temperature_name]  # q first: its dims
  das, datas, perms, dtype = _operands(dataset, names)
  q = das[0]
  if pressure_name not in dataset.coords:
    raise KeyError(pressure_name)
  pcoord = dataset.coords[pressure_name]
  pvalues = np.asarray(pcoord.values)
  if len(pcoord.dims) > 1:
    raise ValueError(f'pressure coordinate {pressure_name!r} has dims '
                     f'{pcoord.dims}: relative humidity takes a scalar or '
                     'one-dimensional pressure coordinate')
  if pcoord.dims and pcoord.dims[0] not in q.dims:
    raise ValueError(f'pressure coordinate {pressure_name!r} lies along '
                     f'{pcoord.dims[0]!r}, which {specific_humidity_name!r} '
                     'lacks; relative humidity does not broadcast it')
  if pvalues.dtype.kind not in 'iuf':
    raise TypeError(f'pressure coordinate {pressure_name!r} has dtype '
                    f'{pvalues.dtype}')
  out_dtype = np.result_type(pvalues.dtype, dtype)
  if out_dtype not in (np.float32, np.float64):
    raise TypeError(f'pressure coordinate {pressure_name!r} of dtype '
                    f'{pvalues.dtype} promotes the result to {out_dtype}')
  dims = q.dims
  shape = tuple(q.sizes[d] for d in dims)
  if pcoord.dims:
    nouter, npres, ninner = _split(shape, dims.index(pcoord.dims[0]))
  else:
    nouter, npres, ninner = 1, 1, int(np.prod(shape, dtype=np.int64))
  pressure = pvalues.astype(np.float64).reshape(-1)
  code = _lib.F64 if dtype == np.float64 else _lib.F32
  out_code = _lib.F64 if out_dtype == np.float64 else _lib.F32
  ctx = _lib.default_context()

  def call(ptrs, out):
    ctx.relative_humidity(code, out_code, ptrs[1], ptrs[0], nouter, npres,
                          ninner, pressure, out[0])

  data, = _streamed.run_whole(datas, [(shape, out_dtype)], call,
                              perms=perms, dtype=dtype)
  coords = dict(das[1].coords)
  coords.update(q.coords)
  if pressure_name not in coords:
    coords[pressure_name] = pcoord
  return xl.DataArray(data, dims, coords)


@dataclasses.dataclass
class LapseRate(dv.DerivedVariable):
  """Lapse rate in temperature, dT/dp / dz/dp with z = Z / 9.81
  (derived_variables.py:341-362).  Needs a `level` dimension and coordinate
  with at least 2 levels."""

  temperature_name: str = 'temperature'
  geopotential_name: str = 'geopotential'

  @property
  def base_variables(self) -> list[str]:
    return [self.temperature_name, self.geopotential_name]

  @property
  def core_dims(self) -> t.Tuple[t.Tuple[t.List[str], ...], t.List[str]]:
    return (['level'], ['level']), ['level']

  def compute(self, dataset):
    return lapse_rate(dataset, self.temperature_name, self.geopotential_name)


@dataclasses.dataclass
class RelativeHumidity(dv.DerivedVariable):
  """Relative humidity from specific humidity (derived_variables.py:433-468),
  MetPy's relative_humidity_from_specific_humidity with Bolton's (1980)
  saturation vapour pressure 6.112 exp(17.67 T / (T + 243.5)), T in degrees
  Celsius.  Temperature is in K and the pressure coordinate in hPa."""

  temperature_name: str = 'temperature'
  specific_humidity_name: str = 'specific_humidity'
  pressure_name: str = 'level'

  @property
  def base_variables(self) -> list[str]:
    return [
        self.temperature_name,
        self.specific_humidity_name,
        self.pressure_name,
    ]

  @property
  def core_dims(self) -> t.Tuple[t.Tuple[t.List[str], ...], t.List[str]]:
    return ([], []), []

  def compute(self, dataset):
    return relative_humidity(dataset, self.temperature_name,
                             self.specific_humidity_name, self.pressure_name)

"""Precipitation accumulations over lead time -- same classes as
weatherbench2/derived_variables.py:471-528 and 685-720.
`PrecipitationAccumulation` runs csrc/precip_accumulation.cu;
`AggregatePrecipitationAccumulation` is the rolling sum of
weatherbench2_b200.resampling (csrc/resample.cu).  Imported into
`weatherbench2_b200.derived_variables`.

CUDA input gives a CUDA tensor of the same dtype on the same device, which the
metric kernels read in place; NumPy, memmap or lazily gathered input is
streamed through the device in bands and gives NumPy.  The result keeps the
input's dims and coords.  Numerics and deviations: include/wb2b200.h and
DESIGN.md section 8e.
"""
from __future__ import annotations

import dataclasses

import numpy as np

from weatherbench2_b200 import _streamed
from weatherbench2_b200 import derived_variables as dv
from weatherbench2_b200 import resampling
from weatherbench2_b200 import xarray_lite as xl


def _lead_values(ds, da: xl.DataArray, lead: str) -> np.ndarray:
  if lead in da.coords:
    return np.asarray(da.coords[lead].values)
  if lead in ds.coords:
    return np.asarray(ds.coords[lead].values)
  raise ValueError(f'{da.name!r} has no {lead!r} coordinate')


def precip_accumulation(da: xl.DataArray, lead: str, window: int,
                        clamp_negative: bool):
  """wb2_precip_accumulation of `da` along `lead`: a CUDA tensor for CUDA
  data, else NumPy streamed within resampling.STREAM_BUDGET_BYTES."""
  if da.dtype not in (np.float32, np.float64):
    raise TypeError(f'variable {da.name!r} has dtype {da.dtype}: precipitation '
                    'accumulation takes float32 or float64 data')
  li = da.dims.index(lead)
  shape = da.shape
  nouter = int(np.prod(shape[:li], dtype=np.int64))
  ntime = shape[li]
  ninner = int(np.prod(shape[li + 1:], dtype=np.int64))
  return _streamed.run('precip_accumulation', da.data,
                       (nouter, ntime, ninner, window, clamp_negative),
                       [(shape, da.dtype)], resampling.STREAM_BUDGET_BYTES)[0]


@dataclasses.dataclass
class PrecipitationAccumulation(dv.DerivedVariable):
  """Precipitation accumulated over the `accumulation_hours` leading up to and
  including each lead time, from a cumulative series
  (derived_variables.py:471-528): tp.diff(lead) summed over a rolling window
  of accumulation_hours / step differences, negative sums set to 0 when
  `set_negative_to_zero`, and a NaN first step, so the output has the input's
  length and dims.

  Errors: AssertionError('All time steps must be equal.') and
  AssertionError('Accumulation time must be multiple of timestep.') as in the
  reference (raised explicitly); ValueError for a missing lead dimension or
  coordinate, a lead axis shorter than 2, a zero or negative step or a window
  below 1 step; TypeError for data other than float32 / float64."""

  total_precipitation_name: str
  accumulation_hours: int
  lead_time_name: str = 'prediction_timedelta'
  set_negative_to_zero: bool = True

  @property
  def base_variables(self) -> list[str]:
    return [self.total_precipitation_name]

  @property
  def core_dims(self):
    return ([self.lead_time_name],), [self.lead_time_name]

  def window(self, lead_values) -> int:
    """Differences per window: accumulation_hours / the lead step."""
    lead = np.asarray(lead_values)
    if lead.ndim != 1 or lead.size < 2:
      raise ValueError(f'{self.lead_time_name!r} needs at least 2 steps '
                       f'(got {lead.size})')
    timestep = np.diff(lead)
    if not np.all(timestep == timestep[0]):
      raise AssertionError('All time steps must be equal.')
    timestep = timestep[0]
    if not timestep > timestep * 0:
      raise ValueError(f'the {self.lead_time_name!r} step must be positive '
                       f'(got {timestep})')
    steps = float(np.timedelta64(self.accumulation_hours, 'h') / timestep)
    if not steps.is_integer():
      raise AssertionError('Accumulation time must be multiple of timestep.')
    if steps < 1:
      raise ValueError(f'accumulation_hours={self.accumulation_hours} gives '
                       f'a window of {int(steps)} steps')
    return int(steps)

  def compute(self, dataset):
    da = dataset[self.total_precipitation_name]
    if self.lead_time_name not in da.dims:
      raise ValueError(f'{self.total_precipitation_name!r} has no '
                       f'{self.lead_time_name!r} dimension')
    w = self.window(_lead_values(dataset, da, self.lead_time_name))
    values = precip_accumulation(da, self.lead_time_name, w,
                                 self.set_negative_to_zero)
    return xl.DataArray(values, da.dims, da.coords, da.name, da.attrs)


@dataclasses.dataclass
class AggregatePrecipitationAccumulation(dv.DerivedVariable):
  """Longer accumulations from shorter ones (derived_variables.py:685-720): a
  rolling sum of `raw_accumulation_name` over accumulation_hours /
  raw_accumulation_hours lead steps, NaN for the first w-1 steps and wherever
  the window holds a NaN (all NaN when w exceeds the lead axis).  No clamp and
  no check of the lead coordinate, as in the reference."""

  accumulation_hours: int
  raw_accumulation_name: str = 'total_precipitation_6hr'
  raw_accumulation_hours: int = 6
  lead_time_name: str = 'prediction_timedelta'

  @property
  def base_variables(self):
    return [self.raw_accumulation_name]

  @property
  def core_dims(self):
    return ([self.lead_time_name],), [self.lead_time_name]

  def compute(self, dataset):
    da = dataset[self.raw_accumulation_name]
    steps = float(np.timedelta64(self.accumulation_hours, 'h') /
                  np.timedelta64(self.raw_accumulation_hours, 'h'))
    if not steps.is_integer():
      raise AssertionError('Accumulation time must be multiple of timestep.')
    if steps < 1:
      raise ValueError(f'accumulation_hours={self.accumulation_hours} gives '
                       f'a window of {int(steps)} steps')
    if self.lead_time_name not in da.dims:
      raise ValueError(f'{self.raw_accumulation_name!r} has no '
                       f'{self.lead_time_name!r} dimension')
    values = resampling._stats(da, self.lead_time_name, ['sum'], skipna=False,  # pylint: disable=protected-access
                               window=int(steps))['sum']
    return xl.DataArray(values, da.dims, da.coords, da.name, da.attrs)

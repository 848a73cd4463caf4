"""A stand-in for the `xarray` package, used ONLY by tests (xarray itself is not
installable here: no network).  It implements exactly the constructor and
attribute surface that weatherbench2_b200.xarray_lite.from_xarray / to_xarray
touch -- the same surface the real package offers -- so the conversion at the
public boundary (Metric.compute_chunk etc. called with xr.Dataset arguments,
weatherbench2/metrics.py:88-115) can be driven end to end.
"""
import numpy as np

__version__ = '0.0-fake'


class _Coord:

  def __init__(self, dims, values, attrs=None):
    self.dims = tuple(dims)
    self.values = np.asarray(values)
    self.attrs = dict(attrs or {})


def _coords(coords, default_dims=None):
  out = {}
  for k, v in (coords or {}).items():
    if isinstance(v, _Coord):
      out[k] = v
    elif isinstance(v, tuple):
      dims = (v[0],) if isinstance(v[0], str) else tuple(v[0])
      out[k] = _Coord(dims, v[1], v[2] if len(v) > 2 else None)
    else:
      v = np.asarray(v)
      out[k] = _Coord((k,) if v.ndim == 1 else (), v)
  return out


class DataArray:

  def __init__(self, data, dims=None, coords=None, name=None, attrs=None):
    self.data = np.asarray(data)
    self.dims = tuple(dims or ())
    self.coords = _coords(coords)
    self.name = name
    self.attrs = dict(attrs or {})

  @property
  def values(self):
    return self.data

  @property
  def shape(self):
    return self.data.shape


class Dataset:

  def __init__(self, data_vars=None, coords=None, attrs=None):
    self.coords = _coords(coords)
    self.attrs = dict(attrs or {})
    self.data_vars = {}
    for k, v in (data_vars or {}).items():
      if isinstance(v, DataArray):
        self.data_vars[k] = v
      else:
        dims, data = v[0], v[1]
        dims = (dims,) if isinstance(dims, str) else tuple(dims)
        cs = {c: cc for c, cc in self.coords.items()
              if all(d in dims for d in cc.dims)}
        self.data_vars[k] = DataArray(data, dims, cs, k,
                                      v[2] if len(v) > 2 else None)

  def __getitem__(self, k):
    return self.data_vars[k]


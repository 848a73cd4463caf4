"""A minimal named-dimension array container (DataArray / Dataset).

WeatherBench2's operator API is written against xarray (`xr.Dataset` in,
`xr.Dataset` out: weatherbench2/metrics.py:88-115).  xarray is not installed on
the build or GPU boxes, so the drop-in operators of this package work on this
small stand-in, which implements exactly the subset of the xarray API the hot
path and its callers use: named dims, coordinate lookup, broadcasting
arithmetic by dimension name, `mean(dim, skipna)`, `isel/sel`, `expand_dims`,
`concat`, `merge`.  The public entry points also take real xarray objects:
`boundary` converts them on the way in and the result on the way out.

`data` may be a NumPy array (host) or a `torch.Tensor` on a CUDA device; the
metric operators read it in place either way.  Everything the container itself
computes (results are tiny) is NumPy.
"""
from __future__ import annotations

import functools
import numbers
from typing import Any, Iterable, Mapping, Optional, Sequence

import numpy as np


def _is_torch(x) -> bool:
  return type(x).__module__.startswith('torch') and hasattr(x, 'data_ptr')


def _np(x) -> np.ndarray:
  if _is_torch(x):
    return x.detach().cpu().numpy()
  return np.asarray(x)


class DataArray:
  """N-d array with named dimensions and coordinates."""

  __array_priority__ = 60

  def __init__(self, data, dims: Optional[Sequence[str]] = None,
               coords: Optional[Mapping[str, Any]] = None,
               name: Optional[str] = None, attrs: Optional[dict] = None):
    if not _is_torch(data):
      data = np.asarray(data)
    if dims is None:
      if data.ndim != 0:
        if coords is not None and len(coords) == data.ndim:
          dims = tuple(coords.keys())
        else:
          raise ValueError('dims are required for non-scalar data')
      else:
        dims = ()
    if isinstance(dims, str):
      dims = (dims,)
    dims = tuple(dims)
    if len(dims) != data.ndim:
      raise ValueError(f'dims {dims} do not match data.ndim={data.ndim}')
    self._data = data
    self.dims = dims
    self.name = name
    self.attrs = dict(attrs or {})
    self.coords: dict[str, 'Coord'] = {}
    for k, v in (coords or {}).items():
      self._set_coord(k, v)

  # -- coords -----------------------------------------------------------------
  def _set_coord(self, k, v):
    if isinstance(v, Coord):
      c = v
    elif isinstance(v, DataArray):
      c = Coord(v.dims, v.values, v.attrs)
    elif isinstance(v, tuple) and len(v) in (2, 3) and (
        isinstance(v[0], (str, tuple, list))):
      d = (v[0],) if isinstance(v[0], str) else tuple(v[0])
      c = Coord(d, np.asarray(v[1]), v[2] if len(v) == 3 else None)
    else:
      a = np.asarray(v)
      c = Coord((k,) if a.ndim == 1 else (), a)
    for d, n in zip(c.dims, c.values.shape):
      if d in self.dims and self.sizes[d] != n:
        raise ValueError(
            f'coord {k!r} has size {n} along {d!r}, data has {self.sizes[d]}')
    if all(d in self.dims for d in c.dims):
      self.coords[k] = c

  # -- basic properties -------------------------------------------------------
  @property
  def data(self):
    return self._data

  @property
  def values(self) -> np.ndarray:
    return _np(self._data)

  @property
  def shape(self):
    return tuple(self._data.shape)

  @property
  def ndim(self):
    return len(self.dims)

  @property
  def dtype(self):
    return self.values.dtype if not _is_torch(self._data) else np.dtype(
        str(self._data.dtype).replace('torch.', ''))

  @property
  def size(self):
    return int(np.prod(self.shape)) if self.shape else 1

  @property
  def sizes(self) -> dict:
    return dict(zip(self.dims, self.shape))

  @property
  def nbytes(self):
    return self.size * self.dtype.itemsize

  def __len__(self):
    return self.shape[0]

  def __array__(self, dtype=None, copy=None):
    v = self.values
    return v.astype(dtype) if dtype is not None else v

  def __float__(self):
    return float(self.values)

  def item(self):
    return self.values.item()

  def __getattr__(self, name):
    # coordinate access as attribute (ds.latitude), like xarray
    if name.startswith('_') or name in ('dims', 'coords', 'attrs', 'name'):
      raise AttributeError(name)
    coords = self.__dict__.get('coords', {})
    if name in coords:
      return self._coord_da(name)
    attrs = self.__dict__.get('attrs', {})
    if name in attrs:
      return attrs[name]
    raise AttributeError(name)

  def _coord_da(self, name) -> 'DataArray':
    c = self.coords[name]
    sub = {k: v for k, v in self.coords.items()
           if all(d in c.dims for d in v.dims)}
    return DataArray(c.values, c.dims, sub, name=name, attrs=c.attrs)

  def __getitem__(self, key):
    if isinstance(key, str):
      return self._coord_da(key)
    if not isinstance(key, tuple):
      key = (key,)
    return self.isel({d: k for d, k in zip(self.dims, key)})

  def __repr__(self):
    return (f'<wb2 DataArray {self.name!r} {self.sizes} '
            f'coords={list(self.coords)}>\n{self.values!r}')

  # -- construction helpers ---------------------------------------------------
  def _replace(self, data, dims=None, coords=None) -> 'DataArray':
    dims = self.dims if dims is None else tuple(dims)
    if coords is None:
      coords = {k: c for k, c in self.coords.items()
                if all(d in dims for d in c.dims)}
    return DataArray(data, dims, coords, self.name, self.attrs)

  def copy(self, data=None, deep=True) -> 'DataArray':
    if data is None:
      data = self._data.clone() if _is_torch(self._data) else (
          self._data.copy() if deep else self._data)
    return self._replace(data)

  def astype(self, dtype) -> 'DataArray':
    return self._replace(self.values.astype(dtype))

  def rename(self, mapping=None, **kw) -> 'DataArray':
    if isinstance(mapping, str) or mapping is None and not kw:
      out = self._replace(self._data)
      out.name = mapping
      return out
    m = dict(mapping or {}, **kw)
    dims = tuple(m.get(d, d) for d in self.dims)
    coords = {m.get(k, k): Coord(tuple(m.get(d, d) for d in c.dims), c.values,
                                 c.attrs) for k, c in self.coords.items()}
    return DataArray(self._data, dims, coords, self.name, self.attrs)

  def assign_coords(self, coords=None, **kw) -> 'DataArray':
    out = self._replace(self._data)
    for k, v in dict(coords or {}, **kw).items():
      out._set_coord(k, v)
    return out

  def assign_attrs(self, *args, **kw) -> 'DataArray':
    out = self._replace(self._data)
    out.attrs.update(*args, **kw)
    return out

  def drop_vars(self, names, errors='raise') -> 'DataArray':
    names = [names] if isinstance(names, str) else list(names)
    out = self._replace(self._data)
    for n in names:
      out.coords.pop(n, None)
    return out

  # -- indexing ---------------------------------------------------------------
  def isel(self, indexers=None, drop=False, **kw) -> 'DataArray':
    idx = dict(indexers or {}, **kw)
    key = []
    new_dims = []
    for d in self.dims:
      k = idx.get(d, slice(None))
      if isinstance(k, DataArray):
        k = k.values
      if isinstance(k, (list, tuple)):
        k = np.asarray(k)
      if isinstance(k, np.ndarray) and k.ndim == 0:
        k = int(k)
      key.append(k)
      if not isinstance(k, numbers.Integral):
        new_dims.append(d)
    data = self._data
    # apply one axis at a time (orthogonal indexing, like xarray)
    for ax in range(len(self.dims) - 1, -1, -1):
      k = key[ax]
      if isinstance(k, slice) and k == slice(None):
        continue
      sl = [slice(None)] * data.ndim
      sl[ax] = k
      data = data[tuple(sl)]
    coords = self._isel_coords(key, drop)
    return DataArray(data, tuple(new_dims), coords, self.name, self.attrs)

  def _isel_coords(self, key, drop=False) -> dict:
    """Coordinates after indexing dimension i of `self.dims` with key[i]."""
    coords = {}
    for name, c in self.coords.items():
      ck = tuple(key[self.dims.index(d)] for d in c.dims)
      v = c.values
      for ax in range(len(c.dims) - 1, -1, -1):
        if isinstance(ck[ax], slice) and ck[ax] == slice(None):
          continue
        sl = [slice(None)] * v.ndim
        sl[ax] = ck[ax]
        v = v[tuple(sl)]
      cd = tuple(d for d, kk in zip(c.dims, ck)
                 if not isinstance(kk, numbers.Integral))
      if drop and not cd and any(
          isinstance(kk, numbers.Integral) for kk in ck):
        continue
      coords[name] = Coord(cd, v, c.attrs)
    return coords

  def _label_indexer(self, dim, label, method=None):
    if dim not in self.coords:
      raise KeyError(f'no coordinate for dimension {dim!r}')
    coord = self.coords[dim].values
    if isinstance(label, slice):
      return label_slice_indices(coord, label)
    if isinstance(label, DataArray):
      label = label.values
    lab = np.asarray(label)
    if lab.ndim == 0:
      return int(_lookup(coord, lab[None], method)[0])
    return _lookup(coord, lab.ravel(), method).reshape(lab.shape)

  def sel(self, indexers=None, method=None, drop=False, **kw) -> 'DataArray':
    idx = dict(indexers or {}, **kw)
    out = self
    for d, label in idx.items():
      if d not in out.dims:
        raise KeyError(d)
      if isinstance(label, DataArray) and label.ndim > 1:
        out = out._vectorized_sel(d, label, method)
        continue
      ind = out._label_indexer(d, label, method)
      if (isinstance(label, slice) and d not in ('latitude', 'longitude') and
          ind.size and (np.diff(ind) == 1).all()):
        # a contiguous label range of an outer dimension stays a VIEW (same
        # strides, shifted base) instead of a fancy-index copy of the data
        ind = slice(int(ind[0]), int(ind[-1]) + 1)
      if isinstance(label, DataArray) and label.ndim == 1 and (
          label.dims[0] != d):
        out = out._vectorized_sel(d, label, method)
        continue
      out = out.isel({d: ind}, drop=drop)
    return out

  def _vectorized_sel(self, dim, label: 'DataArray', method=None):
    """`.sel(dim=<N-d DataArray>)`: `dim` is replaced by the indexer's dims
    (the by-init gather truth.sel(time=forecast.valid_time),
    weatherbench2/evaluation.py:475)."""
    coord = self.coords[dim].values
    ind = _lookup(coord, label.values.ravel(), method).reshape(label.shape)
    ax = self.dims.index(dim)
    data = np.take(self.values, ind, axis=ax)  # inserts label dims at `ax`
    dims = self.dims[:ax] + label.dims + self.dims[ax + 1:]
    coords = {k: c for k, c in self.coords.items() if dim not in c.dims}
    for k, c in label.coords.items():
      coords.setdefault(k, c)
    coords[dim] = Coord(label.dims, label.values)
    return DataArray(data, dims, coords, self.name, self.attrs)

  # -- shape manipulation -----------------------------------------------------
  def transpose(self, *dims) -> 'DataArray':
    if not dims:
      dims = self.dims[::-1]
    if Ellipsis in dims:
      i = dims.index(Ellipsis)
      rest = tuple(d for d in self.dims if d not in dims)
      dims = dims[:i] + rest + dims[i + 1:]
    dims = tuple(d for d in dims if d in self.dims)
    perm = [self.dims.index(d) for d in dims]
    data = (self._data.permute(*perm) if _is_torch(self._data)
            else np.transpose(self._data, perm))
    return self._replace(data, dims)

  def expand_dims(self, dim=None, axis=0, **kw) -> 'DataArray':
    if isinstance(dim, str):
      dim = {dim: 1}
    elif isinstance(dim, (list, tuple)):
      dim = {d: 1 for d in dim}
    dim = dict(dim or {}, **kw)
    out = self
    for name, val in reversed(list(dim.items())):
      if isinstance(val, DataArray):
        val = val.values
      if isinstance(val, numbers.Integral):
        n, cvals = int(val), None
      else:
        cvals = np.asarray(val)
        n = cvals.size
      v = out.values
      data = np.broadcast_to(v[None], (n,) + v.shape)
      coords = dict(out.coords)
      if cvals is not None:
        coords[name] = Coord((name,), cvals.reshape(-1))
      elif name in coords and not coords[name].dims:
        c = coords[name]
        coords[name] = Coord((name,), np.broadcast_to(c.values, (n,)).copy())
      out = DataArray(data, (name,) + out.dims, coords, out.name, out.attrs)
    return out

  def squeeze(self, dim=None, drop=False) -> 'DataArray':
    dims = [d for d, n in self.sizes.items() if n == 1] if dim is None else (
        [dim] if isinstance(dim, str) else list(dim))
    return self.isel({d: 0 for d in dims}, drop=drop)

  # -- reductions -------------------------------------------------------------
  def _reduce(self, fn_skip, fn, dim, skipna) -> 'DataArray':
    import warnings
    if dim is None:
      axes = tuple(range(self.ndim))
      dims_left = ()
    else:
      red = [dim] if isinstance(dim, str) else list(dim)
      axes = tuple(self.dims.index(d) for d in red)
      dims_left = tuple(d for d in self.dims if d not in red)
    v = self.values
    with warnings.catch_warnings():
      warnings.simplefilter('ignore', RuntimeWarning)
      with np.errstate(invalid='ignore', divide='ignore'):
        use_skip = skipna or (skipna is None and v.dtype.kind == 'f')
        r = fn_skip(v, axis=axes) if use_skip else fn(v, axis=axes)
    return self._replace(np.asarray(r), dims_left)

  def mean(self, dim=None, skipna=None, **kw) -> 'DataArray':
    return self._reduce(np.nanmean, np.mean, dim, skipna)

  def sum(self, dim=None, skipna=None, **kw) -> 'DataArray':
    return self._reduce(np.nansum, np.sum, dim, skipna)

  def max(self, dim=None, skipna=None, **kw) -> 'DataArray':
    return self._reduce(np.nanmax, np.max, dim, skipna)

  def min(self, dim=None, skipna=None, **kw) -> 'DataArray':
    return self._reduce(np.nanmin, np.min, dim, skipna)

  def diff(self, dim) -> 'DataArray':
    ax = self.dims.index(dim)
    coords = {k: (Coord(c.dims, np.take(
        c.values, np.arange(1, c.values.shape[c.dims.index(dim)]),
        axis=c.dims.index(dim)), c.attrs) if dim in c.dims else c)
              for k, c in self.coords.items()}
    return DataArray(np.diff(self.values, axis=ax), self.dims, coords,
                     self.name, self.attrs)

  def all(self):
    return bool(np.all(self.values))

  def any(self):
    return bool(np.any(self.values))

  def isnull(self):
    return self._replace(np.isnan(self.values))

  def notnull(self):
    return self._replace(~np.isnan(self.values))

  def where(self, cond, other=np.nan):
    a, c, dims, coords = _broadcast(self, cond)
    if isinstance(other, DataArray):
      _, o, _, _ = _broadcast(self, other)
    else:
      o = other
    return DataArray(np.where(c, a, o), dims, coords, self.name, self.attrs)

  def fillna(self, value):
    v = self.values
    return self._replace(np.where(np.isnan(v), value, v))

  def equals(self, other) -> bool:
    return (isinstance(other, DataArray) and self.dims == other.dims and
            self.shape == other.shape and
            np.array_equal(self.values, other.values, equal_nan=True))

  # -- arithmetic -------------------------------------------------------------
  def _binary(self, other, op, reflexive=False):
    if isinstance(other, Dataset):
      return NotImplemented
    a, b, dims, coords = _broadcast(self, other)
    with np.errstate(invalid='ignore', divide='ignore', over='ignore'):
      r = op(b, a) if reflexive else op(a, b)
    return DataArray(r, dims, coords, self.name)

  def __add__(self, o): return self._binary(o, np.add)
  def __radd__(self, o): return self._binary(o, np.add, True)
  def __sub__(self, o): return self._binary(o, np.subtract)
  def __rsub__(self, o): return self._binary(o, np.subtract, True)
  def __mul__(self, o): return self._binary(o, np.multiply)
  def __rmul__(self, o): return self._binary(o, np.multiply, True)
  def __truediv__(self, o): return self._binary(o, np.divide)
  def __rtruediv__(self, o): return self._binary(o, np.divide, True)
  def __pow__(self, o): return self._binary(o, np.power)
  def __lt__(self, o): return self._binary(o, np.less)
  def __le__(self, o): return self._binary(o, np.less_equal)
  def __gt__(self, o): return self._binary(o, np.greater)
  def __ge__(self, o): return self._binary(o, np.greater_equal)
  def __neg__(self): return self._replace(-self.values)
  def __abs__(self): return self._replace(np.abs(self.values))

  def __array_ufunc__(self, ufunc, method, *inputs, **kwargs):
    if method != '__call__' or kwargs.get('out') is not None:
      return NotImplemented
    if len(inputs) == 1:
      with np.errstate(invalid='ignore', divide='ignore'):
        return self._replace(ufunc(self.values, **kwargs))
    if len(inputs) == 2:
      x, y = inputs
      if isinstance(x, Dataset) or isinstance(y, Dataset):
        return NotImplemented
      if x is self:
        return self._binary(y, ufunc)
      return self._binary(x, ufunc, reflexive=True)
    return NotImplemented


class Coord:
  """A coordinate variable: (dims, values, attrs)."""
  __slots__ = ('dims', 'values', 'attrs')

  def __init__(self, dims, values, attrs=None):
    self.dims = tuple(dims)
    self.values = np.asarray(values)
    self.attrs = dict(attrs or {})


def label_slice_indices(coord: np.ndarray, s: slice) -> np.ndarray:
  """Positions selected by `.sel(dim=slice(lo, hi))` on a monotonic increasing
  index: pandas `slice_indexer`, BOTH ends inclusive
  (weatherbench2/regions.py:79-84 relies on it)."""
  coord = np.asarray(coord)
  if s.step is not None:
    raise ValueError('label slices with a step are not supported')
  if coord.size > 1 and not (np.diff(coord.astype(np.float64)) > 0).all():
    if (np.diff(coord.astype(np.float64)) < 0).all():
      rev = label_slice_indices(
          coord[::-1], slice(s.stop, s.start))
      return (coord.size - 1 - rev)[::-1]
    raise KeyError('label slicing needs a monotonic coordinate')
  start = 0 if s.start is None else int(np.searchsorted(coord, s.start, 'left'))
  stop = coord.size if s.stop is None else int(
      np.searchsorted(coord, s.stop, 'right'))
  return np.arange(start, max(start, stop))


def _lookup(coord: np.ndarray, labels: np.ndarray, method=None) -> np.ndarray:
  coord = np.asarray(coord)
  labels = np.asarray(labels)
  if coord.dtype.kind in 'mM' or labels.dtype.kind in 'mM':
    unit = 'ns'
    kind = coord.dtype.kind if coord.dtype.kind in 'mM' else labels.dtype.kind
    t = 'datetime64[ns]' if kind == 'M' else 'timedelta64[ns]'
    coord = coord.astype(t).astype(np.int64)
    labels = labels.astype(t).astype(np.int64)
    del unit
  if method == 'nearest':
    return np.abs(coord[None, :].astype(np.float64) -
                  labels[:, None].astype(np.float64)).argmin(axis=1)
  order = np.argsort(coord, kind='stable')
  pos = np.searchsorted(coord[order], labels)
  pos = np.clip(pos, 0, coord.size - 1)
  idx = order[pos]
  bad = coord[idx] != labels
  if bad.any():
    raise KeyError(f'labels not found in coordinate: {labels[bad][:5]}')
  return idx


def _broadcast(a: DataArray, b):
  """xarray arithmetic broadcasting: dims of `a`, then new dims of `b`."""
  av = a.values
  if isinstance(b, (bool, int, float, complex)):
    # a Python scalar stays "weak" (NEP 50): float32 data compared with /
    # scaled by 0.25e-3 stays float32, as under xarray; np.asarray(scalar)
    # would be a float64 0-d ARRAY and promote the whole operation
    return av, b, a.dims, dict(a.coords)
  if not isinstance(b, DataArray):
    bv = _np(b)
    if bv.ndim not in (0,) and bv.shape != av.shape:
      raise ValueError('cannot broadcast a bare ndarray against a DataArray')
    return av, bv, a.dims, dict(a.coords)
  dims = list(a.dims) + [d for d in b.dims if d not in a.dims]
  for d in b.dims:
    if d in a.dims and a.sizes[d] != b.sizes[d]:
      raise ValueError(
          f'size mismatch along {d!r}: {a.sizes[d]} vs {b.sizes[d]}')

  def expand(x: DataArray):
    perm = [x.dims.index(d) for d in dims if d in x.dims]
    v = np.transpose(x.values, perm)
    return v[tuple(slice(None) if d in x.dims else None for d in dims)]

  coords = dict(b.coords)
  coords.update(a.coords)
  return expand(a), expand(b), tuple(dims), coords


class Dataset:
  """Dict of DataArrays sharing coordinates."""

  __array_priority__ = 70

  def __init__(self, data_vars: Optional[Mapping[str, Any]] = None,
               coords: Optional[Mapping[str, Any]] = None,
               attrs: Optional[dict] = None):
    self._vars: dict[str, DataArray] = {}
    self._coords: dict[str, Coord] = {}
    self.attrs = dict(attrs or {})
    for k, v in (coords or {}).items():
      if isinstance(v, Coord):
        self._coords[k] = v
      elif isinstance(v, DataArray):
        self._coords[k] = Coord(v.dims, v.values, v.attrs)
      elif isinstance(v, tuple) and len(v) in (2, 3) and isinstance(
          v[0], (str, tuple, list)):
        d = (v[0],) if isinstance(v[0], str) else tuple(v[0])
        self._coords[k] = Coord(d, np.asarray(v[1]),
                                v[2] if len(v) == 3 else None)
      else:
        a = np.asarray(v)
        self._coords[k] = Coord((k,) if a.ndim == 1 else (), a)
    for k, v in (data_vars or {}).items():
      self[k] = v

  # -- mapping ----------------------------------------------------------------
  def __setitem__(self, key, value):
    if isinstance(value, DataArray):
      da = value
    elif isinstance(value, tuple):
      da = DataArray(value[1], value[0],
                     attrs=value[2] if len(value) > 2 else None)
    else:
      da = DataArray(value)
    for k, c in da.coords.items():
      self._coords.setdefault(k, c)
    if hasattr(da, 'lazy_source'):  # keep lazily gathered views lazy
      da.name = key
      self._vars[key] = da
      return
    coords = {k: c for k, c in self._coords.items()
              if all(d in da.dims for d in c.dims)}
    self._vars[key] = DataArray(da.data, da.dims, coords, key, da.attrs)

  def __getitem__(self, key):
    if isinstance(key, str):
      if key in self._vars:
        v = self._vars[key]
        if hasattr(v, 'lazy_source'):
          return v
        coords = {k: c for k, c in self._coords.items()
                  if all(d in v.dims for d in c.dims)}
        return DataArray(v.data, v.dims, coords, key, v.attrs)
      if key in self._coords:
        c = self._coords[key]
        sub = {k: v for k, v in self._coords.items()
               if all(d in c.dims for d in v.dims)}
        return DataArray(c.values, c.dims, sub, key, c.attrs)
      raise KeyError(key)
    # a coordinate name may be listed, as in xarray: it stays a coordinate
    # (RelativeHumidity lists its pressure coordinate among its base variables)
    missing = [k for k in key if k not in self._vars and k not in self._coords]
    if missing:
      raise KeyError(missing)
    return Dataset({k: self[k] for k in key if k in self._vars}, self._coords,
                   self.attrs)

  def __getattr__(self, name):
    if name.startswith('_') or name == 'attrs':
      raise AttributeError(name)
    d = self.__dict__
    if name in d.get('_vars', {}) or name in d.get('_coords', {}):
      return self[name]
    if name in d.get('attrs', {}):
      return d['attrs'][name]
    raise AttributeError(name)

  def __contains__(self, k):
    return k in self._vars or k in self._coords

  def __iter__(self):
    return iter(self._vars)

  def __len__(self):
    return len(self._vars)

  def keys(self):
    return self._vars.keys()

  def values(self):
    return [self[k] for k in self._vars]

  def items(self):
    return [(k, self[k]) for k in self._vars]

  @property
  def data_vars(self):
    return {k: self[k] for k in self._vars}

  @property
  def coords(self):
    return self._coords

  @property
  def sizes(self) -> dict:
    out = {}
    for v in self._vars.values():
      out.update(v.sizes)
    for c in self._coords.values():
      for d, n in zip(c.dims, c.values.shape):
        out.setdefault(d, n)
    return out

  @property
  def dims(self):
    return self.sizes

  @property
  def nbytes(self):
    return sum(v.nbytes for v in self._vars.values())

  def __repr__(self):
    lines = [f'<wb2 Dataset sizes={self.sizes} attrs={self.attrs}>']
    for k, v in self._vars.items():
      lines.append(f'  {k} {v.dims} {v.dtype}')
    return '\n'.join(lines)

  # -- functional helpers -----------------------------------------------------
  def _map(self, fn, keep_attrs=True) -> 'Dataset':
    out = Dataset(coords=None, attrs=self.attrs if keep_attrs else None)
    res = {k: fn(self[k]) for k in self._vars}
    # coordinates that survive on any variable, plus scalar coords
    keep = {}
    all_dims = set()
    for v in res.values():
      all_dims.update(v.dims)
      keep.update(v.coords)
    for k, c in self._coords.items():
      if k not in keep and all(d in all_dims for d in c.dims) and (
          not res or not self._vars):
        keep[k] = c
    out._coords = dict(keep)
    for k, v in res.items():
      out[k] = v
    return out

  def copy(self, data=None, deep=True) -> 'Dataset':
    if data is None:
      return self._map(lambda v: v.copy(deep=deep))
    out = Dataset(coords=self._coords, attrs=self.attrs)
    for k in self._vars:
      out[k] = self[k]._replace(data[k])
    return out

  def mean(self, dim=None, skipna=None, **kw):
    return self._map(
        lambda v: v.mean(_present(dim, v), skipna) if _present(dim, v) != ()
        or dim is None else v)

  def sum(self, dim=None, skipna=None, **kw):
    return self._map(
        lambda v: v.sum(_present(dim, v), skipna) if _present(dim, v) != ()
        or dim is None else v)

  def isel(self, indexers=None, drop=False, **kw):
    idx = dict(indexers or {}, **kw)
    out = self._map(lambda v: v.isel(
        {d: k for d, k in idx.items() if d in v.dims}, drop=drop))
    # coords not attached to any variable
    holder = DataArray(np.zeros(()), ())
    for k, c in self._coords.items():
      if k not in out._coords:
        tmp = DataArray(np.zeros(c.values.shape), c.dims, {k: c})
        sub = tmp.isel({d: kk for d, kk in idx.items() if d in c.dims},
                       drop=drop)
        if k in sub.coords:
          out._coords[k] = sub.coords[k]
    del holder
    return out

  def sel(self, indexers=None, method=None, drop=False, **kw):
    idx = dict(indexers or {}, **kw)
    return self._map(lambda v: v.sel(
        {d: k for d, k in idx.items() if d in v.dims}, method=method,
        drop=drop))

  def transpose(self, *dims):
    return self._map(lambda v: v.transpose(*dims))

  def expand_dims(self, dim=None, **kw):
    return self._map(lambda v: v.expand_dims(dim, **kw))

  def rename(self, mapping=None, **kw):
    m = dict(mapping or {}, **kw)
    out = Dataset(attrs=self.attrs)
    out._coords = {m.get(k, k): Coord(tuple(m.get(d, d) for d in c.dims),
                                      c.values, c.attrs)
                   for k, c in self._coords.items()}
    for k in self._vars:
      v = self[k]
      out[m.get(k, k)] = v.rename({d: m[d] for d in v.dims if d in m} or None
                                  ) if any(d in m for d in v.dims) else v
    return out

  def rename_vars(self, mapping):
    return self.rename(mapping)

  def assign_coords(self, coords=None, **kw):
    out = self._map(lambda v: v)
    for k, v in dict(coords or {}, **kw).items():
      tmp = Dataset(coords={k: v})
      out._coords[k] = tmp._coords[k]
    return out

  def assign_attrs(self, *args, **kw):
    out = self._map(lambda v: v)
    out.attrs = dict(self.attrs)
    out.attrs.update(*args, **kw)
    return out

  def drop_vars(self, names, errors='raise'):
    names = [names] if isinstance(names, str) else list(names)
    out = Dataset(attrs=self.attrs)
    out._coords = {k: c for k, c in self._coords.items() if k not in names}
    for k in self._vars:
      if k not in names:
        out[k] = self[k].drop_vars(names)
    return out

  def equals(self, other) -> bool:
    return (isinstance(other, Dataset) and set(self._vars) == set(other._vars)
            and all(self[k].equals(other[k]) for k in self._vars))

  # -- arithmetic (inner join on data variables, like xarray) -----------------
  def _binary(self, other, op, reflexive=False):
    out = Dataset(attrs=None)
    if isinstance(other, Dataset):
      keys = [k for k in self._vars if k in other._vars]
      pairs = {k: (self[k], other[k]) for k in keys}
    else:
      pairs = {k: (self[k], other) for k in self._vars}
    for k, (a, b) in pairs.items():
      r = a._binary(b, op, reflexive) if isinstance(a, DataArray) else None
      out[k] = r
    for k, c in self._coords.items():
      if not c.dims:
        out._coords.setdefault(k, c)
    return out

  def __add__(self, o): return self._binary(o, np.add)
  def __radd__(self, o): return self._binary(o, np.add, True)
  def __sub__(self, o): return self._binary(o, np.subtract)
  def __rsub__(self, o): return self._binary(o, np.subtract, True)
  def __mul__(self, o): return self._binary(o, np.multiply)
  def __rmul__(self, o): return self._binary(o, np.multiply, True)
  def __truediv__(self, o): return self._binary(o, np.divide)
  def __rtruediv__(self, o): return self._binary(o, np.divide, True)
  def __pow__(self, o): return self._binary(o, np.power)
  def __neg__(self): return self._map(lambda v: -v)
  def __abs__(self): return self._map(abs)

  def __array_ufunc__(self, ufunc, method, *inputs, **kwargs):
    if method != '__call__':
      return NotImplemented
    if len(inputs) == 1:
      return self._map(lambda v: ufunc(v, **kwargs))
    if len(inputs) == 2:
      x, y = inputs
      if x is self:
        return self._binary(y, ufunc)
      return self._binary(x, ufunc, reflexive=True)
    return NotImplemented


def _present(dim, v: DataArray):
  if dim is None:
    return None
  dims = [dim] if isinstance(dim, str) else list(dim)
  return tuple(d for d in dims if d in v.dims)


# -- module-level functions (xr.concat / xr.merge / xr.zeros_like) -------------
def zeros_like(obj):
  if isinstance(obj, Dataset):
    return obj._map(zeros_like)
  return obj._replace(np.zeros_like(obj.values))


def concat(objs: Sequence, dim: str):
  objs = list(objs)
  if isinstance(objs[0], Dataset):
    keys = list(objs[0].keys())
    out = Dataset(attrs=objs[0].attrs)
    for k in keys:
      out[k] = concat([o[k] for o in objs], dim)
    return out
  first = objs[0]
  if dim in first.dims:
    ax = first.dims.index(dim)
    data = np.concatenate([o.transpose(*first.dims).values for o in objs],
                          axis=ax)
    dims = first.dims
  else:
    data = np.stack([o.transpose(*first.dims).values for o in objs], axis=0)
    dims = (dim,) + first.dims
  coords = {k: c for k, c in first.coords.items() if dim not in c.dims}
  if all(dim in o.coords for o in objs):
    coords[dim] = Coord((dim,), np.concatenate(
        [np.atleast_1d(o.coords[dim].values) for o in objs]))
  return DataArray(data, dims, coords, first.name, first.attrs)


def merge(objs: Iterable) -> Dataset:
  """xr.merge for results that differ along 1-D dimension coordinates
  (weatherbench2/evaluation.py:437 merges per-metric results along `metric`):
  outer join on every dimension coordinate, NaN fill."""
  objs = [o if isinstance(o, Dataset) else Dataset({o.name: o}) for o in objs]
  # union of index coordinates, in order of first appearance
  index = {}
  for o in objs:
    for k, c in o.coords.items():
      if c.dims == (k,):
        cur = index.setdefault(k, [])
        for v in c.values.tolist():
          if v not in cur:
            cur.append(v)
  out = Dataset()
  for o in objs:
    for k, c in o.coords.items():
      if c.dims != (k,):
        out._coords.setdefault(k, c)
  for k, vals in index.items():
    first = next(o.coords[k].values for o in objs if k in o.coords)
    out._coords[k] = Coord((k,), np.asarray(vals, dtype=first.dtype))
  names = []
  for o in objs:
    for k in o.keys():
      if k not in names:
        names.append(k)
  for name in names:
    parts = [o[name] for o in objs if name in o.keys()]
    dims = parts[0].dims
    shape = tuple(len(index[d]) if d in index else parts[0].sizes[d]
                  for d in dims)
    full = np.full(shape, np.nan, dtype=np.result_type(
        parts[0].values.dtype, np.float32))
    for p in parts:
      p = p.transpose(*dims)
      sel = []
      for d in dims:
        if d in index and d in p.coords:
          sel.append(np.asarray(
              [index[d].index(v) for v in p.coords[d].values.tolist()]))
        else:
          sel.append(np.arange(p.sizes[d]))
      full[np.ix_(*sel)] = p.values
    coords = {k: c for k, c in out._coords.items()
              if all(d in dims for d in c.dims)}
    out[name] = DataArray(full, dims, coords, name, parts[0].attrs)
  return out


# -- conversion to / from real xarray (only when it is importable) -------------
def have_xarray() -> bool:
  try:
    import xarray  # pylint: disable=unused-import,import-outside-toplevel
    return True
  except Exception:  # pylint: disable=broad-except
    return False


def from_xarray(obj):
  """xr.Dataset / xr.DataArray -> lite container (no copy of the data)."""
  if isinstance(obj, (Dataset, DataArray)) or obj is None:
    return obj
  if not is_native_xarray(obj):
    return obj  # plain arrays etc. pass through
  import xarray as xr  # pylint: disable=import-outside-toplevel
  if isinstance(obj, xr.DataArray):
    coords = {k: Coord(tuple(v.dims), v.values, dict(v.attrs))
              for k, v in obj.coords.items()}
    return DataArray(obj.data if isinstance(obj.data, np.ndarray) else
                     obj.values, tuple(obj.dims), coords, obj.name,
                     dict(obj.attrs))
  coords = {k: Coord(tuple(v.dims), v.values, dict(v.attrs))
            for k, v in obj.coords.items()}
  return Dataset({k: (tuple(v.dims), v.data if isinstance(v.data, np.ndarray)
                      else v.values, dict(v.attrs))
                  for k, v in obj.data_vars.items()}, coords, dict(obj.attrs))


def to_xarray(obj):
  import xarray as xr  # pylint: disable=import-outside-toplevel
  if isinstance(obj, DataArray):
    return xr.DataArray(obj.values, dims=obj.dims, coords={
        k: (c.dims, c.values, c.attrs) for k, c in obj.coords.items()},
                        name=obj.name, attrs=obj.attrs)
  return xr.Dataset({k: (v.dims, v.values, v.attrs) for k, v in obj.items()},
                    coords={k: (c.dims, c.values, c.attrs)
                            for k, c in obj.coords.items()}, attrs=obj.attrs)


def is_native_xarray(obj) -> bool:
  return type(obj).__module__.startswith('xarray')


def _lite(obj):
  return from_xarray(obj) if is_native_xarray(obj) else obj


def boundary(fn):
  """Lets `fn`, written for lite containers, take native xarray objects too.

  Every native argument, positional or keyword, is converted with
  `from_xarray` before the call.  If the first container argument (native or
  lite) was native, a lite Dataset or DataArray result is converted with
  `to_xarray`; any other result passes through.  A call with lite arguments
  converts nothing, so operators that call each other convert only at the
  outermost call."""

  @functools.wraps(fn)
  def call(*args, **kwargs):
    values = args + tuple(kwargs.values())
    if not any(is_native_xarray(a) for a in values):
      return fn(*args, **kwargs)
    first = next(a for a in values
                 if isinstance(a, (Dataset, DataArray)) or is_native_xarray(a))
    out = fn(*map(_lite, args), **{k: _lite(v) for k, v in kwargs.items()})
    if is_native_xarray(first) and isinstance(out, (Dataset, DataArray)):
      return to_xarray(out)
    return out

  return call


class Boundary:
  """Base class that puts `boundary` on the methods named in
  `_boundary_methods`, in the class that names them and in every subclass
  that overrides one."""

  _boundary_methods: tuple = ()

  def __init_subclass__(cls, **kwargs):
    super().__init_subclass__(**kwargs)
    for name in cls._boundary_methods:
      if name in cls.__dict__:
        setattr(cls, name, boundary(cls.__dict__[name]))


class LazyGather(DataArray):
  """A DataArray view `source.isel(dim=positions)` with N-d positions, not
  materialised unless `.values` is read.  `_spatial.prepare_operand` turns it
  into offset-table addressing."""

  def __init__(self, source: DataArray, index_maps: dict,
               extra_coords: Optional[dict] = None):
    dims, shape = [], []
    for d, n in source.sizes.items():
      if d in index_maps:
        tdims, pos = index_maps[d]
        for td, tn in zip(tdims, np.asarray(pos).shape):
          if td not in dims:
            dims.append(td)
            shape.append(tn)
      else:
        dims.append(d)
        shape.append(n)
    self._source = source
    self._index_maps = {d: (tuple(td), np.asarray(p, dtype=np.int64))
                        for d, (td, p) in index_maps.items()}
    self._lazy_dims = tuple(dims)
    self._lazy_shape = tuple(shape)
    self._materialised = None
    self.dims = tuple(dims)
    self.name = source.name
    self.attrs = dict(source.attrs)
    self.coords = {k: c for k, c in source.coords.items()
                   if not any(d in index_maps for d in c.dims)}
    for k, c in (extra_coords or {}).items():
      self.coords[k] = c

  @property
  def lazy_source(self):
    return self._source, self._index_maps

  @property
  def shape(self):
    return self._lazy_shape

  @property
  def _data(self):
    if self._materialised is None:
      # xarray's vectorised indexing: indexers that share dimensions are
      # applied POINTWISE along them (the day-of-year / hour lookup of one
      # valid time), not as an outer product.
      v = self._source.values
      sdims = list(self._source.dims)
      mapped = [d for d in sdims if d in self._index_maps]
      jdims, jshape = [], []
      for d in mapped:
        tdims, pos = self._index_maps[d]
        for td, tn in zip(tdims, pos.shape):
          if td not in jdims:
            jdims.append(td)
            jshape.append(tn)
      rest = [d for d in sdims if d not in self._index_maps]
      v = np.transpose(v, [sdims.index(d) for d in mapped + rest])
      index = []
      for d in mapped:
        tdims, pos = self._index_maps[d]
        p = np.transpose(pos, [tdims.index(td) for td in jdims if td in tdims])
        p = p[tuple(slice(None) if td in tdims else None for td in jdims)]
        index.append(np.broadcast_to(p, jshape))
      v = v[tuple(index)] if index else v
      have = jdims + rest
      perm = [have.index(d) for d in self._lazy_dims]
      self._materialised = np.transpose(v, perm)
    return self._materialised

  @_data.setter
  def _data(self, value):  # DataArray.__init__ is bypassed
    self._materialised = value

  @property
  def dtype(self):
    return self._source.dtype

  def isel(self, indexers=None, drop=False, **kw) -> 'DataArray':
    """Slices / index arrays keep the view lazy: a looked-up dimension
    restricts the position tables, any other one the source (chunking a
    climatological or persistence forecast along init_time must not
    materialise the forecast-sized copy).  Integer indexers fall back to the
    materialised array."""
    idx = dict(indexers or {}, **kw)
    norm = {}
    for d, k in idx.items():
      if d not in self.dims:
        continue
      if isinstance(k, DataArray):
        k = k.values
      if isinstance(k, (list, tuple)):
        k = np.asarray(k)
      if not (isinstance(k, slice) or (isinstance(k, np.ndarray) and
                                       k.ndim == 1)):
        return DataArray(self.values, self.dims, self.coords, self.name,
                         self.attrs).isel(idx, drop=drop)
      norm[d] = k
    source, maps = self._source, dict(self._index_maps)
    for d, k in norm.items():
      looked_up = False
      for sd, (tdims, pos) in list(maps.items()):
        if d in tdims:
          sl = [slice(None)] * pos.ndim
          sl[tdims.index(d)] = k
          maps[sd] = (tdims, pos[tuple(sl)])
          looked_up = True
      if not looked_up:
        if isinstance(k, slice):
          source = source.isel({d: k})  # a view of the source
        else:
          # picking labels of an untouched dimension becomes one more lookup:
          # nothing of the (possibly very long) source record is copied
          maps[d] = ((d,), np.asarray(k, dtype=np.int64))
    key = [norm.get(d, slice(None)) for d in self.dims]
    coords = self._isel_coords(key, drop)
    out = LazyGather(source, maps)
    out.coords = coords
    out.name, out.attrs = self.name, dict(self.attrs)
    return out


def align_inner(a: DataArray, b: DataArray):
  """xarray's default arithmetic alignment (join='inner') of two arrays along
  the dimensions they share: labels present in both, in the order of `a`.
  Returns the inputs untouched when the shared coordinates already agree;
  otherwise lazily gathered views (no data copied)."""
  maps_a, maps_b = {}, {}
  for d in a.dims:
    if d not in b.dims or d not in a.coords or d not in b.coords:
      continue
    ca, cb = a.coords[d].values, b.coords[d].values
    if ca.shape == cb.shape and np.array_equal(ca, cb):
      continue
    if d in ('latitude', 'longitude'):
      # the kernels address whole (lat, lon) slabs: a label join along a
      # spatial dimension cannot be folded into an offset table, and silently
      # falling back to positional alignment would be wrong (the reference's
      # _ensure_aligned_grid makes the grids identical up front)
      raise ValueError(
          f'{d} coordinates of the two operands differ; align the grids first '
          '(evaluation.open_forecast_and_truth_datasets assigns the '
          "forecast's coordinates like the reference's _ensure_aligned_grid)")
    keep = np.isin(ca, cb)
    labels = ca[keep]
    maps_a[d] = ((d,), np.nonzero(keep)[0])
    maps_b[d] = ((d,), _lookup(cb, labels))
  if not maps_a:
    return a, b

  def view(x, maps):
    if hasattr(x, 'lazy_source'):
      # already a gathered view (a by-init truth, a climatological or
      # persistence forecast): restrict its position tables, stay lazy
      return x.isel({d: pos for d, (_, pos) in maps.items()})
    extra = {d: Coord((d,), x.coords[d].values[pos])
             for d, (_, pos) in maps.items()}
    return LazyGather(x, maps, extra_coords=extra)

  return view(a, maps_a), view(b, maps_b)

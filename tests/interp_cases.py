"""Seeded bilinear, nearest-neighbour and spectrum-interpolation cases with
their expected values (K8: csrc/regrid_interp.cu; csrc/preprocess.cu
wb2_spectrum_interp).

Bilinear.  The reference interpolates with `jnp.interp` in float32, latitude
first, then longitude.  `jnp_interp` below is a literal float32 transcription
of it: `x % period` (jnp.remainder: fmod plus the sign fix, -0.0 stays -0.0),
the stable key sort, the extended axis, searchsorted(side='right'), the clip,
`dx0 = |dx| <= spacing(eps)`, `fp[i-1] + (delta / dx) * df`, and the trailing
`where`s for left and right.  Given the host's taps the kernel is bit-equal to
it, NaN and inf included (NaN payloads aside: the GPU's arithmetic NaN is
canonical).  `bilinear_float64` repeats the two lerps in float64 with the
model's float32 fractions; per cell, with u = 2^-24 and the float64 values,
    lerp error  <= u |a + t (b - a)| + 2.01 u |t (b - a)|
and the longitude lerp adds its own to the larger of its two inputs' bounds
(t is in [0, 1]), so `bilinear_bound` is that sum, times 1.01.

Nearest.  The expected indices come from a BallTree (haversine) over the
meshgrid of (latitude, longitude) in radians, raveled -- independently of the
host's `nearest_neighbor_indices`.

Spectrum interpolation.  The expected value is the installed scipy's
`interp1d(kind='linear', bounds_error=False)` per latitude row, as the oracle
computes it (float64 weights times the float32 spectrum, so the result is
float64).  `scipy_weighted` transcribes its interval choice and formula;
`spectrum_bound` is 1 float32 ulp of the exact value plus the float64 error of
that formula (6 u64 of |w_hi y_hi| + |w_lo y_lo|).
"""
import dataclasses
import functools

import numpy as np

F32 = np.float32
U32 = 2.0 ** -24
U64 = 2.0 ** -53
EPS_SPACING = np.spacing(np.finfo(F32).eps)  # jnp.interp's dx0 threshold

# the branches a target coordinate can take through jnp.interp
BRANCHES = ('lerp', 'node', 'left', 'right', 'dx0', 'wrap', 'one_lon')


# ---- jnp.interp in float32 -----------------------------------------------------
def jnp_remainder(x, p):
  r = np.fmod(x, p)
  return np.where((r != 0) & ((r < 0) != (p < 0)), r + p, r).astype(x.dtype)


def _prepare(x, xp, fp, period, dtype=F32):
  x = np.asarray(x, F32)
  xp = np.asarray(xp, F32)
  fp = np.asarray(fp, dtype)
  if period is not None:
    p = np.abs(F32(period))
    x = jnp_remainder(x, p)
    xp = jnp_remainder(xp, p)
    order = np.argsort(xp, kind='stable')  # lax.sort_key_val is stable
    xp, fp = xp[order], fp[order]
    xp = np.concatenate([xp[-1:] - p, xp, xp[:1] + p]).astype(F32)
    fp = np.concatenate([fp[-1:], fp, fp[:1]])
  i = np.clip(np.searchsorted(xp, x, side='right'), 1, xp.size - 1)
  return x, xp, fp, i


def jnp_interp(x, xp, fp, left=None, right=None, period=None, dtype=F32):
  """jnp.interp along axis 0 of `fp` (the trailing axes are carried along).
  dtype=np.float64 evaluates the same taps and float32 fractions in float64."""
  x, xp, fp, i = _prepare(x, xp, fp, period, dtype)
  sh = (-1,) + (1,) * (fp.ndim - 1)
  dx = (xp[i] - xp[i - 1]).astype(F32)
  delta = (x - xp[i - 1]).astype(F32)
  dx0 = np.abs(dx) <= EPS_SPACING
  t = (delta / np.where(dx0, F32(1), dx)).astype(F32).astype(dtype)
  with np.errstate(invalid='ignore', over='ignore'):
    df = fp[i] - fp[i - 1]
    f = np.where(dx0.reshape(sh), fp[i - 1], fp[i - 1] + t.reshape(sh) * df)
  if period is None:
    f = np.where((x < xp[0]).reshape(sh),
                 fp[0] if left is None else dtype(left), f)
    f = np.where((x > xp[-1]).reshape(sh),
                 fp[-1] if right is None else dtype(right), f)
  return f.astype(dtype)


def jnp_branches(x, xp, period=None):
  """Per target coordinate, the jnp.interp branch it takes (BRANCHES)."""
  xq, xe, _, i = _prepare(x, xp, np.zeros(np.size(xp)), period)
  dx = (xe[i] - xe[i - 1]).astype(F32)
  delta = (xq - xe[i - 1]).astype(F32)
  out = np.where(delta == 0, 'node', 'lerp').astype(object)
  if period is not None:
    out[(i == 1) | (i == xe.size - 1)] = 'wrap'
    if np.size(xp) == 1:
      out[:] = 'one_lon'
  out[np.abs(dx) <= EPS_SPACING] = 'dx0'
  if period is None:
    out[xq < xe[0]] = 'left'
    out[xq > xe[-1]] = 'right'
  return out


def _lat_lon_kw(src):
  lat = {} if src.includes_poles else dict(left=np.nan, right=np.nan)
  lon = dict(period=360) if src.periodic else dict(left=np.nan, right=np.nan)
  return lat, lon


def _two_pass(fields, src, tgt, interp):
  """(nf, nlon, nlat) -> (nf, nlon_t, nlat_t), latitude first."""
  lat_kw, lon_kw = _lat_lon_kw(src)
  y = interp(tgt.latitudes, src.latitudes, np.moveaxis(fields, -1, 0), **lat_kw)
  y = interp(tgt.longitudes, src.longitudes, np.moveaxis(y, -1, 0), **lon_kw)
  return np.moveaxis(y, -1, 0)  # (nlon_t, nlat_t, nf) -> (nf, nlon_t, nlat_t)


def bilinear_model(fields, src, tgt):
  return _two_pass(fields, src, tgt, jnp_interp)


def bilinear_lon_first(fields, src, tgt):
  """Mutant: longitude first, then latitude."""
  lat_kw, lon_kw = _lat_lon_kw(src)
  y = jnp_interp(tgt.longitudes, src.longitudes, np.swapaxes(fields, 0, 1),
                 **lon_kw)                                   # (nlon_t, nf, nlat)
  y = jnp_interp(tgt.latitudes, src.latitudes, np.moveaxis(y, -1, 0), **lat_kw)
  return np.transpose(y, (2, 1, 0))  # (nlat_t, nlon_t, nf) -> (nf, ...)


def bilinear_fma(fields, src, tgt):
  """Mutant: each lerp fused into one rounding (a + t * d in float64, then
  float32)."""
  def interp(x, xp, fp, **kw):
    x_, xp_, fp_, i = _prepare(x, xp, fp, kw.get('period'))
    sh = (-1,) + (1,) * (fp_.ndim - 1)
    t = ((x_ - xp_[i - 1]) / (xp_[i] - xp_[i - 1])).astype(F32)
    with np.errstate(invalid='ignore', over='ignore'):
      d = (fp_[i] - fp_[i - 1]).astype(F32)
      f = (fp_[i - 1].astype(np.float64) + t.reshape(sh).astype(np.float64) *
           d.astype(np.float64)).astype(F32)
    exact = jnp_interp(x, xp, fp, **kw)
    keep = (np.abs(xp_[i] - xp_[i - 1]) <= EPS_SPACING)
    if kw.get('period') is None:
      keep = keep | (x_ < xp_[0]) | (x_ > xp_[-1])
    return np.where(keep.reshape(sh), exact, f)
  return _two_pass(fields, src, tgt, interp)


def bilinear_float64(fields, src, tgt):
  return _two_pass(fields, src, tgt,
                   functools.partial(jnp_interp, dtype=np.float64))


def bilinear_bound(fields, src, tgt):
  """Per-cell bound of the float32 model against bilinear_float64."""
  lat_kw, lon_kw = _lat_lon_kw(src)

  def lerp_err(x, xp, fp, e_in, kw):
    xq, xe, fpe, i = _prepare(x, xp, fp, kw.get('period'), np.float64)
    _, _, ee, _ = _prepare(x, xp, e_in, kw.get('period'), np.float64)
    sh = (-1,) + (1,) * (fpe.ndim - 1)
    dx = (xe[i] - xe[i - 1]).astype(F32)
    t = ((xq - xe[i - 1]).astype(F32) /
         np.where(np.abs(dx) <= EPS_SPACING, F32(1), dx)).astype(F32)
    with np.errstate(invalid='ignore'):
      td = np.abs(t.astype(np.float64).reshape(sh) * (fpe[i] - fpe[i - 1]))
      val = np.abs(fpe[i - 1] + t.astype(np.float64).reshape(sh) *
                   (fpe[i] - fpe[i - 1]))
      e = U32 * (val + 2.01 * td) + np.maximum(ee[i], ee[i - 1])
    # the `where` branches return a tap: its bound, nothing added
    e = np.where((np.abs(dx) <= EPS_SPACING).reshape(sh), ee[i - 1], e)
    if kw.get('period') is None:
      e = np.where((xq < xe[0]).reshape(sh), ee[0], e)
      e = np.where((xq > xe[-1]).reshape(sh), ee[-1], e)
    return e

  f64 = np.asarray(fields, np.float64)
  e0 = np.zeros_like(f64)
  y = jnp_interp(tgt.latitudes, src.latitudes, np.moveaxis(f64, -1, 0),
                 dtype=np.float64, **lat_kw)
  ey = lerp_err(tgt.latitudes, src.latitudes, np.moveaxis(f64, -1, 0),
                np.moveaxis(e0, -1, 0), lat_kw)
  e = lerp_err(tgt.longitudes, src.longitudes, np.moveaxis(y, -1, 0),
               np.moveaxis(ey, -1, 0), lon_kw)
  return 1.01 * np.moveaxis(e, -1, 0)


def kernel_formula(fields, lon_taps, lat_taps):
  """The kernel's arithmetic on the host's taps, in float32: i0 = -1 NaN,
  t < 0 fp[i0] itself, else a + t * (b - a) with three roundings."""
  def lerp(a, i0, i1, t, axis):
    i0, i1 = np.asarray(i0), np.asarray(i1)
    lo = np.take(a, np.maximum(i0, 0), axis=axis)
    hi = np.take(a, np.maximum(i1, 0), axis=axis)
    sh = [1] * a.ndim
    sh[axis] = -1
    with np.errstate(invalid='ignore', over='ignore'):
      v = (lo + np.asarray(t, F32).reshape(sh) * (hi - lo)).astype(F32)
    v = np.where(np.asarray(t).reshape(sh) < 0, lo, v)
    return np.where((i0 < 0).reshape(sh), F32(np.nan), v).astype(F32)
  y = lerp(np.asarray(fields, F32), *lat_taps, axis=-1)
  return lerp(y, *lon_taps, axis=-2)


# ---- nearest ---------------------------------------------------------------------
def ball_tree_indices(src, tgt):
  from sklearn.neighbors import BallTree  # pylint: disable=import-outside-toplevel

  def mesh(grid):
    lat, lon = np.meshgrid(np.deg2rad(np.asarray(grid.latitudes, np.float64)),
                           np.deg2rad(np.asarray(grid.longitudes, np.float64)))
    return np.stack([lat.ravel(), lon.ravel()], axis=-1)
  tree = BallTree(mesh(src), metric='haversine')
  return tree.query(mesh(tgt), return_distance=False)[:, 0]


# ---- grids and fields ----------------------------------------------------------------
@dataclasses.dataclass(frozen=True)
class GridSpec:
  longitudes: np.ndarray
  latitudes: np.ndarray
  periodic: bool = True
  includes_poles: bool = True

  @property
  def shape(self):
    return (len(self.longitudes), len(self.latitudes))

  def grid(self):
    from weatherbench2_b200 import regridding as rg  # pylint: disable=import-outside-toplevel
    return rg.Grid(longitudes=np.asarray(self.longitudes),
                   latitudes=np.asarray(self.latitudes),
                   periodic=self.periodic, includes_poles=self.includes_poles)


def equiangular(nlon, nlat, poles=True, **kw):
  edge = 90.0 if poles else 90.0 - 90.0 / nlat
  return GridSpec(np.linspace(0, 360, nlon, endpoint=False),
                  np.linspace(-edge, edge, nlat), includes_poles=poles, **kw)


def realistic_fields(shape, seed):
  """z500, temperature, surface pressure, specific humidity, u wind,
  precipitation with exact zeros, SST with land NaN -- (7, nlon, nlat)."""
  rs = np.random.RandomState(seed)
  nlon, nlat = shape
  lon = np.linspace(0, 2 * np.pi, nlon, endpoint=False)[:, None]
  lat = np.linspace(-np.pi / 2, np.pi / 2, nlat)[None, :]
  noise = lambda s: s * rs.standard_normal(shape)  # noqa: E731
  z500 = 54000 + 3000 * np.cos(lat) ** 2 + 600 * np.sin(4 * lon) * np.cos(lat)
  temp = 230 + 60 * np.cos(lat) + noise(2)
  sp = 101325 - 8000 * (rs.uniform(size=shape) > 0.8) + noise(300)
  q = np.exp(rs.uniform(np.log(1e-5), np.log(2e-2), shape))
  u = 50 * np.tanh(noise(1.0)) * np.cos(lat)
  precip = np.where(rs.uniform(size=shape) < 0.6, 0.0,
                    rs.exponential(2e-3, shape))
  sst = np.where(rs.uniform(size=shape) < 0.3, np.nan,
                 271.4 + 30 * np.cos(lat) + noise(0.5))
  return np.stack([z500 + noise(20), temp, sp, q, u, precip, sst]).astype(F32)


def structural_fields(shape, seed):
  """A constant (exact everywhere), a -0.0 / 0.0 checkerboard, spikes at the
  seam, the poles and the first and last rows, and NaN / +-inf on the end
  latitude rows (the clamped and NaN-outside branches), at the seam and
  inside."""
  rs = np.random.RandomState(seed)
  nlon, nlat = shape
  const = np.full(shape, 287.25)
  zeros = np.where((np.arange(nlon)[:, None] + np.arange(nlat)) % 2, 0.0, -0.0)
  spikes = rs.uniform(-1, 1, shape)
  for a, c in ((0, 0), (nlon - 1, nlat - 1), (0, nlat // 2), (nlon - 1, 0),
               (nlon // 2, 0), (nlon // 2, nlat - 1)):
    spikes[a, c] = 5e4
  special = 1000 + rs.standard_normal(shape)
  # first and last latitude rows (the clamped and NaN-outside taps): inf, -inf
  # and NaN on alternating longitudes, so an infinity survives a longitude
  # lerp as its right tap (a + t * (inf - a) = inf for t > 0)
  special[1::4, 0] = np.inf
  special[2::4, -1] = -np.inf
  special[3::4, 0] = np.nan
  special[-1, nlat // 2] = np.inf    # the seam
  special[0, nlat // 3] = np.nan
  special[nlon // 2, nlat // 2] = np.nan
  if nlat > 2:
    special[nlon // 3, 1] = -np.inf
  return np.stack([const, zeros, spikes, special]).astype(F32)


@dataclasses.dataclass(frozen=True)
class BilinearCase:
  name: str
  src: GridSpec
  tgt: GridSpec
  realistic: bool   # realistic fields as well as the structural ones
  lat_branches: frozenset
  lon_branches: frozenset
  seed: int = 0

  @functools.cached_property
  def fields(self):
    parts = [structural_fields(self.src.shape, self.seed)]
    if self.realistic:
      parts.insert(0, realistic_fields(self.src.shape, self.seed + 1))
    return np.concatenate(parts)

  @property
  def nreal(self):
    return 7 if self.realistic else 0


def _b(*names):
  return frozenset(names)


def bilinear_cases():
  e025 = equiangular(1440, 721)
  e15 = equiangular(240, 121)
  g64 = equiangular(64, 32, poles=False)
  shift = GridSpec(e15.longitudes + 0.75, (e15.latitudes[:-1] + 0.75))
  centred = GridSpec(np.array([-0.0, -180.0, -90.25, -1e-6, 0.0, 44.9,
                               179.75, 359.99, 360.0, 359.75]),
                     np.linspace(-87.5, 87.5, 8))
  seam = GridSpec(np.linspace(0, 360, 37), np.linspace(-90, 90, 19))
  seam_t = GridSpec(np.array([0.0, 5.0, 355.0, 359.0, 360.0, -5.0]),
                    np.linspace(-85, 85, 7))
  lam = GridSpec(np.linspace(10, 60, 21), np.linspace(20, 50, 13),
                 periodic=False, includes_poles=False)
  lam_t = GridSpec(np.array([0.0, 10.0, 12.3, 59.9, 60.0, 70.0]),
                   np.array([10.0, 20.0, 33.3, 50.0, 55.0]))
  no_poles = equiangular(72, 36, poles=False)
  poles_t = GridSpec(np.linspace(0, 355, 72), np.array([-90.0, -88.0, 0.0,
                                                        88.0, 90.0]))
  short = GridSpec(np.linspace(0, 350, 36), np.linspace(-60, 60, 13))
  short_t = GridSpec(np.linspace(0, 355, 72), np.linspace(-90, 90, 19))
  one_lat = GridSpec(np.linspace(0, 350, 36), np.array([10.0]))
  one_lat_t = GridSpec(np.linspace(0, 355, 72), np.array([-20.0, 10.0, 40.0]))
  one_lon = GridSpec(np.array([0.0]), np.linspace(-90, 90, 19))
  one_lon_t = GridSpec(np.array([0.0, 45.0, 200.0]), np.linspace(-90, 90, 37))
  tiny = GridSpec(np.array([0.0, 1e-15, 90.0, 180.0]),
                  np.array([-1e-15, 0.0, 45.0]))
  tiny_t = GridSpec(np.array([5e-16, 45.0]),
                    np.array([-5e-16, 0.0, 30.0, 60.0]))
  return [
      BilinearCase('era5_025_to_15', e025, e15, True,
                   _b('node', 'lerp'), _b('node')),
      BilinearCase('era5_025_to_64x32', e025, g64, True,
                   _b('lerp'), _b('lerp', 'node')),
      BilinearCase('upsample_15_to_025', e15, e025, True,
                   _b('node', 'lerp'), _b('node', 'lerp', 'wrap')),
      BilinearCase('identity_15', e15, e15, True, _b('node'), _b('node')),
      BilinearCase('half_cell_shift', e15, shift, True, _b('lerp'),
                   _b('lerp', 'wrap')),
      BilinearCase('centred_targets', e15, centred, False, _b('lerp'),
                   _b('node', 'lerp', 'wrap')),
      BilinearCase('duplicate_seam', seam, seam_t, False, _b('lerp'),
                   _b('node', 'lerp')),
      BilinearCase('limited_area', lam, lam_t, True, _b('left', 'right', 'node',
                                                        'lerp'),
                   _b('left', 'right', 'node', 'lerp')),
      BilinearCase('pole_targets_no_poles', no_poles, poles_t, False,
                   _b('left', 'right', 'lerp'), _b('node', 'wrap')),
      BilinearCase('clamped_short_poles', short, short_t, False,
                   _b('left', 'right', 'node', 'lerp'), _b('node', 'lerp',
                                                           'wrap')),
      BilinearCase('single_latitude', one_lat, one_lat_t, False,
                   _b('left', 'right', 'dx0'), _b('node', 'lerp', 'wrap')),
      BilinearCase('single_longitude', one_lon, one_lon_t, False,
                   _b('node', 'lerp'), _b('one_lon')),
      BilinearCase('tiny_spacing', tiny, tiny_t, False,
                   _b('dx0', 'node', 'lerp', 'right'), _b('dx0', 'lerp')),
  ]


def reached_branches(case):
  lat = set(jnp_branches(case.tgt.latitudes, case.src.latitudes))
  per = 360 if case.src.periodic else None
  lon = set(jnp_branches(case.tgt.longitudes, case.src.longitudes, per))
  if not case.src.periodic:
    lon = {b if b not in ('wrap', 'one_lon') else 'lerp' for b in lon}
  return lat, lon


# ---- spectrum interpolation ------------------------------------------------------------
def frequency_table(nlon, nlat):
  """(nlat, nk) frequencies as ZonalEnergySpectrum.compute makes them at an
  equiangular grid with poles: rfftfreq(nlon) / (circumference * dlon / 360)."""
  from weatherbench2_b200 import derived_variables as dvs  # pylint: disable=import-outside-toplevel
  lat = np.linspace(-90, 90, nlat)
  spacing = (np.cos(lat * np.pi / 180) * 2 * np.pi * dvs.EARTH_RADIUS_M *
             (360 / nlon) / 360)
  return (np.fft.rfftfreq(nlon)[:, None] / spacing[None, :]).T


def default_frequencies(table):
  fv = table.T  # (wavenumber, latitude), as the reference holds it
  return np.linspace(fv.max(axis=1).min(), fv.min(axis=1).max(),
                     num=fv.shape[0])


def spectra(nfield, table, seed):
  """k^-3 spectra from ~1e9 down to ~1e-3 (per-row amplitudes), a row of
  zeros, and NaN / +-inf next to nodes."""
  rs = np.random.RandomState(seed)
  nrow, nk = table.shape
  k = np.arange(nk)
  amp = 10.0 ** rs.uniform(-2, 9, (nfield, nrow, 1))
  s = amp * (1.0 + k) ** -3 * np.exp(0.3 * rs.standard_normal((nfield, nrow,
                                                               nk)))
  s = np.maximum(s, 1e-3 * rs.uniform(0.5, 1, s.shape))
  s[0, 0] = 0.0
  if nk > 4:
    s[:, 1, 2] = np.inf
    s[:, 2, nk // 2] = np.nan
    s[:, 3 % nrow, 0] = -np.inf
    s[:, 3 % nrow, nk - 1] = np.inf
  return s.astype(F32)


@dataclasses.dataclass(frozen=True)
class SpectrumCase:
  name: str
  table: np.ndarray   # (nrow, nk) float64
  freqs: np.ndarray   # float64
  nfield: int
  seed: int = 0

  @functools.cached_property
  def spec(self):
    return spectra(self.nfield, self.table, self.seed)


def spectrum_cases():
  out = []
  for nlon, nlat, nfield in ((1440, 721, 2), (240, 121, 3), (64, 33, 4)):
    tab = frequency_table(nlon, nlat)
    r = nlat // 3
    row = tab[r]
    edges = np.array([np.nextafter(row[0], -np.inf), row[0],
                      np.nextafter(row[0], np.inf),
                      np.nextafter(row[-1], -np.inf), row[-1],
                      np.nextafter(row[-1], np.inf), np.nan, -1.0,
                      tab.max() * 2, np.inf])
    freqs = np.concatenate([default_frequencies(tab), row[1:-1:7],
                            tab[1][2:5], edges])
    out.append(SpectrumCase(f'zonal_{nlon}x{nlat}', tab, freqs, nfield,
                            seed=nlon))
  tab2 = np.array([[0.0, 1.0], [0.5, 2.0], [1e-7, 1e-6]])
  out.append(SpectrumCase('nk2', tab2, np.array([0.0, 0.5, 1.0, 2.0, 0.75,
                                                 5e-7, 1e-6, 3.0, -1.0,
                                                 np.nan]), 3))
  return out


def scipy_reference(case):
  """(nfield, nrow, nf) float64, scipy interp1d per row (the oracle)."""
  from oracle import wb2_oracle as orc  # pylint: disable=import-outside-toplevel
  return orc.interpolate_spectral_frequencies(case.spec, case.table.T,
                                              case.freqs)[0]


def scipy_weighted(case):
  """scipy's _call_linear in float64, transcribed."""
  out = np.empty(case.spec.shape[:2] + (case.freqs.size,))
  f = case.freqs
  for r, x in enumerate(case.table):
    hi = np.clip(np.searchsorted(x, f, side='left'), 1, x.size - 1)
    lo = hi - 1
    w_hi = (f - x[lo]) / (x[hi] - x[lo])
    w_lo = (x[hi] - f) / (x[hi] - x[lo])
    y = case.spec[:, r].astype(np.float64)
    with np.errstate(invalid='ignore'):
      v = w_hi * y[:, hi] + w_lo * y[:, lo]
    v[:, (f < x[0]) | (f > x[-1])] = np.nan
    out[:, r] = v
  return out


def spectrum_bound(case):
  """1 float32 ulp of the value plus 6 u64 (|w_hi y_hi| + |w_lo y_lo|)."""
  out = np.zeros(case.spec.shape[:2] + (case.freqs.size,))
  f = case.freqs
  for r, x in enumerate(case.table):
    hi = np.clip(np.searchsorted(x, f, side='left'), 1, x.size - 1)
    lo = hi - 1
    w_hi = np.abs((f - x[lo]) / (x[hi] - x[lo]))
    w_lo = np.abs((x[hi] - f) / (x[hi] - x[lo]))
    y = np.abs(case.spec[:, r].astype(np.float64))
    with np.errstate(invalid='ignore'):
      s = w_hi * y[:, hi] + w_lo * y[:, lo]
    out[:, r] = 6 * U64 * s
  ref = np.abs(scipy_weighted(case))
  return np.spacing(ref.astype(F32)).astype(np.float64) + out


def exact_spectrum(case):
  """The interpolant in extended precision (np.longdouble where it is wider)."""
  ld = np.longdouble
  out = np.empty(case.spec.shape[:2] + (case.freqs.size,), dtype=ld)
  f = case.freqs.astype(ld)
  for r, x in enumerate(case.table.astype(ld)):
    hi = np.clip(np.searchsorted(x, f, side='left'), 1, x.size - 1)
    lo = hi - 1
    y = case.spec[:, r].astype(ld)
    with np.errstate(invalid='ignore'):
      v = ((f - x[lo]) * y[:, hi] + (x[hi] - f) * y[:, lo]) / (x[hi] - x[lo])
    v[:, (f < x[0]) | (f > x[-1])] = np.nan
    out[:, r] = v
  return out

"""Seeded conservative-regridding cases with float64 answers and a per-cell
error bound (K5: csrc/regrid_tma.cu, csrc/regrid.cu).

Each case holds a longitude and a latitude CSR (built by the package from two
grids, or raw), float32 fields (nfield, nlon_s, nlat_s) and the kernel
instance it claims under the default dispatch: 'TMA G<g> DPT<d> NTAP<n>' or
'LDG DPT<d>'.  `instance()` is a transcription of the host-side eligibility
rule of regrid_tma_try / regrid_tma_launch (base and stride alignment,
nlat_s <= 1024, G * maxtap <= 128, at most two runs of source rows per group,
staging + ybuf + descriptors within 55 KB at G = 2 or 110 KB at G = 4), then
the DPT and the seven-tap specialisation.

Families:
  * realistic: z500 (~5e4 with planetary waves), temperature with a latitude
    gradient, surface pressure with orography-like steps, specific humidity
    1e-8 .. 2e-2, u / v wind, precipitation (mostly exact zeros) and SST with
    land NaN, on the grid pairs users regrid between;
  * structural, on one carrier per instance: zeros, all-NaN, a constant with
    NaN rows and columns (exactly 1 or NaN), isolated spikes with disjoint
    footprints at run heads and tails, the periodic seam, the first and last
    latitude and the last DPT slice;
  * infinite inputs on every carrier: +inf, -inf, both signs in one
    footprint, inf next to NaN;
  * raw CSR for what no grid pair reaches: odd source latitude counts, three
    runs per group, G * maxtap > 128, empty target rows, G = 4 at DPT 1 and
    with seven taps.

The answer is banded: only stored taps contribute, NaN is missing and +-inf
propagate in IEEE arithmetic (`reference`).  Per target cell, with x0 = x
with NaN set to 0 and u = 2^-24,
    T = sum wl w x0,  C = sum wl w [x not NaN],  A = sum wl w |x0|
    |got - T / C| <= u |T / C| + 1.01 (n_a + m_c) u (A + |T|) / C
where n_a and m_c are the longitude and latitude tap counts of the cell
(DESIGN.md K5 derives it)."""
import dataclasses
import functools

import numpy as np
import scipy.sparse as sps

from weatherbench2_b200 import _lib
from weatherbench2_b200 import regridding as rg

U = 2.0 ** -24
GROUP_DESC_BYTES = 64  # sizeof(rgt::GroupDesc)
TAP_BYTES = 8          # sizeof(rgt::Tap)

INSTANCES = (tuple(f'TMA G{g} DPT{d} NTAP0' for g in (2, 4)
                   for d in (1, 2, 3, 4)) +
             ('TMA G2 DPT3 NTAP7', 'TMA G4 DPT3 NTAP7') +
             tuple(f'LDG DPT{d}' for d in (1, 2, 3, 4)))


# ---- CSR --------------------------------------------------------------------
def raw_csr(n_src, rows, nan_rows=()):
  """A CsrSpec from [(cols, vals), ...] as given (no sorting, no checks)."""
  s = _lib.CsrSpec.__new__(_lib.CsrSpec)
  s.n_src, s.n_tgt = int(n_src), len(rows)
  s.row_ptr = np.cumsum([0] + [len(c) for c, _ in rows]).astype(np.int32)
  cols = [np.asarray(c, np.int32) for c, _ in rows]
  vals = [np.asarray(v, np.float32) for _, v in rows]
  s.col_idx = np.concatenate(cols + [np.zeros(1, np.int32)]).astype(np.int32)
  s.val = np.concatenate(vals + [np.zeros(1, np.float32)]).astype(np.float32)
  s.nan_row = np.zeros(len(rows), np.uint8)
  s.nan_row[list(nan_rows)] = 1
  return s


def taps(csr, i):
  lo, hi = csr.row_ptr[i], csr.row_ptr[i + 1]
  return csr.col_idx[lo:hi], csr.val[lo:hi]


def ntaps(csr):
  return np.diff(csr.row_ptr).astype(np.int64)


# ---- path model -------------------------------------------------------------
def _tma_smem(lon, nlat_s, g):
  """Shared memory regrid_tma_launch<g> asks for, or None if not eligible."""
  nt = ntaps(lon)
  maxtap = max(1, int(nt.max()))
  if g * maxtap > 128:
    return None
  stage = 4
  for a0 in range(0, lon.n_tgt, g):
    a1 = min(lon.n_tgt, a0 + g)
    rows = np.unique(lon.col_idx[lon.row_ptr[a0]:lon.row_ptr[a1]])
    runs = []
    for r in rows.tolist():
      if runs and r == runs[-1][1] + 1:
        runs[-1][1] = r
      else:
        runs.append([r, r])
    if len(runs) > 2:
      return None
    used = 0
    for first, last in runs:
      f, e = first * nlat_s, (last + 1) * nlat_s
      used += ((e - (f & ~3)) + 3) & ~3
    stage = max(stage, used)
  return (stage * 4 + g * 2 * nlat_s * 4 + 2 * GROUP_DESC_BYTES +
          2 * g * maxtap * TAP_BYTES + 32)


def instance(lon, lat, src_stride=None, base_offset=0, force_ldg=False):
  """The kernel wb2_regrid_conservative launches: 'TMA G.. DPT.. NTAP..',
  'LDG DPT..' or 'unsupported' (WB2_EUNSUPPORTED)."""
  nlat_s = lat.n_src
  if nlat_s > 1024:
    return 'unsupported'
  src_stride = lon.n_src * nlat_s if src_stride is None else src_stride
  dpt = -(-nlat_s // 256)
  if (not force_ldg and base_offset % 16 == 0 and src_stride % 4 == 0 and
      lon.n_src * nlat_s < 2 ** 31):
    nt = ntaps(lon)
    seven = int(nt.min()) == 7 and int(nt.max()) == 7
    for g, limit in ((2, 55), (4, 110)):
      smem = _tma_smem(lon, nlat_s, g)
      if smem is not None and smem <= limit * 1024:
        return f'TMA G{g} DPT{dpt} NTAP{7 if dpt == 3 and seven else 0}'
  return f'LDG DPT{dpt}'


def ldg_group_rows(lon, g=4):
  """Source rows of each LDG group (the union its dense table covers)."""
  return [np.unique(lon.col_idx[lon.row_ptr[a0]:
                                lon.row_ptr[min(lon.n_tgt, a0 + g)]])
          for a0 in range(0, lon.n_tgt, g)]


# ---- float64 reference and bound --------------------------------------------
def _sparse(csr):
  nnz = int(csr.row_ptr[-1])
  return sps.csr_matrix((csr.val[:nnz].astype(np.float64),
                         csr.col_idx[:nnz].copy(), csr.row_ptr.copy()),
                        shape=(csr.n_tgt, csr.n_src))


def _contract(lon, lat, x):
  """sum_b sum_d Wlon[a,b] Wlat[c,d] x[f,b,d] over stored taps only."""
  nf, nb, nd = x.shape
  y = _sparse(lon) @ x.transpose(1, 0, 2).reshape(nb, nf * nd)  # (a, f*d)
  y = y.reshape(lon.n_tgt, nf, nd).transpose(2, 1, 0).reshape(nd, -1)
  z = _sparse(lat) @ y                                          # (c, f*a)
  return z.reshape(lat.n_tgt, nf, lon.n_tgt).transpose(1, 2, 0)


@dataclasses.dataclass
class Reference:
  want: np.ndarray   # float64 T / C, NaN where the kernels give NaN
  bound: np.ndarray  # per-cell bound (inf where want is not finite)
  T: np.ndarray
  C: np.ndarray
  A: np.ndarray


def reference(lon, lat, x):
  x = np.asarray(x, np.float64)
  ok = ~np.isnan(x)
  x0 = np.where(ok, x, 0.0)
  with np.errstate(invalid='ignore', over='ignore'):
    t = _contract(lon, lat, x0)
    c = _contract(lon, lat, ok.astype(np.float64))
    a = _contract(lon, lat, np.abs(x0))
  with np.errstate(invalid='ignore', divide='ignore'):
    want = t / c
    want[:, lon.nan_row.astype(bool), :] = np.nan
    want[:, :, lat.nan_row.astype(bool)] = np.nan
    k = ntaps(lon)[:, None] + ntaps(lat)[None, :]
    bound = U * np.abs(want) + 1.01 * k * U * (a + np.abs(t)) / c
  bound = np.where(np.isfinite(want), bound, np.inf)
  return Reference(want, bound, t, c, a)


def violations(got, ref, zero_exact=False, value_exact=False):
  """Messages for the cells of `got` (float32) that break the contract:
  NaN / inf pattern and sign, the per-cell bound, and optionally +0 bits where
  the answer is 0 and float32(answer) bit for bit where it is finite."""
  got = np.asarray(got, np.float32)
  want, bound = ref.want, ref.bound
  out = []
  gn, wn = np.isnan(got), np.isnan(want)
  if (gn != wn).any():
    i = np.argwhere(gn != wn)[0]
    out.append(f'NaN pattern: {int((gn != wn).sum())} cells, first {tuple(i)}'
               f' got {got[tuple(i)]} want {want[tuple(i)]}')
  winf = np.isinf(want)
  if (got[winf] != want[winf]).any() or (np.isinf(got) & ~winf).any():
    out.append('inf pattern differs')
  fin = np.isfinite(want)
  with np.errstate(invalid='ignore'):
    err = np.abs(got.astype(np.float64) - want)
  bad = fin & ~(err <= bound)
  if bad.any():
    i = np.argwhere(bad)[0]
    out.append(f'{int(bad.sum())} cells out of bound, first {tuple(i)} got '
               f'{got[tuple(i)]!r} want {want[tuple(i)]!r} err {err[tuple(i)]:.3g}'
               f' bound {bound[tuple(i)]:.3g}')
  if zero_exact:
    z = fin & (want == 0)
    if (got[z].view(np.int32) != 0).any():
      out.append(f'{int((got[z].view(np.int32) != 0).sum())} cells outside '
                 'every footprint are not +0')
  if value_exact and (got[fin] != want[fin].astype(np.float32)).any():
    out.append(f'{int((got[fin] != want[fin].astype(np.float32)).sum())} '
               'cells differ from the exact answer')
  return out


# ---- float32 models of the kernels' tap order -------------------------------
def _fma32(w, x, y):
  # w * x is exact in float64; one rounding to float64, one to float32
  return (w.astype(np.float64) * x + y).astype(np.float32)


def _padded(csr, drop_smallest=False):
  nt = ntaps(csr)
  m = max(1, int(nt.max()))
  idx = np.zeros((csr.n_tgt, m), np.int64)
  w = np.zeros((csr.n_tgt, m), np.float32)
  for i in range(csr.n_tgt):
    c, v = taps(csr, i)
    if drop_smallest and len(c) > 1:
      keep = np.arange(len(c)) != int(np.argmin(v))
      c, v = c[keep], v[keep]
    idx[i, :len(c)], w[i, :len(c)] = c, v
  return idx, w


def model_f32(lon, lat, x, drop_smallest=False):
  """float32 model of regrid_tma_kernel on finite / NaN inputs: each target's
  taps in CSR order through fmaf chains, then one float32 division.  With
  drop_smallest, every longitude target loses its smallest-weight tap."""
  x = np.asarray(x, np.float32)
  ok = ~np.isnan(x)
  x0 = np.where(ok, x, np.float32(0))
  one = ok.astype(np.float32)
  li, lw = _padded(lon, drop_smallest)
  y = np.zeros((x.shape[0], lon.n_tgt, lat.n_src), np.float32)
  v = np.zeros_like(y)
  for j in range(li.shape[1]):  # padding taps have w = 0: fmaf(0, x, y) = y
    wj = lw[:, j][None, :, None]
    y = _fma32(wj, x0[:, li[:, j], :], y)
    v = _fma32(wj, one[:, li[:, j], :], v)
  ti, tw = _padded(lat)
  tot = np.zeros((x.shape[0], lon.n_tgt, lat.n_tgt), np.float32)
  cnt = np.zeros_like(tot)
  for j in range(ti.shape[1]):
    wj = tw[:, j][None, None, :]
    tot = _fma32(wj, y[:, :, ti[:, j]], tot)
    cnt = _fma32(wj, v[:, :, ti[:, j]], cnt)
  with np.errstate(invalid='ignore', divide='ignore'):
    r = tot / cnt
  r[:, lon.nan_row.astype(bool), :] = np.nan
  r[:, :, lat.nan_row.astype(bool)] = np.nan
  return r


# ---- grids and fields -------------------------------------------------------
def lons(n, scheme=rg.LongitudeScheme.START_AT_ZERO):
  return rg.longitude_values(scheme, n)


def lats(n, poles=True):
  return rg.latitude_values(
      rg.LatitudeSpacing.EQUIANGULAR_WITH_POLES if poles else
      rg.LatitudeSpacing.EQUIANGULAR_WITHOUT_POLES, n)


def gaussian_lats(n):
  """Gauss-Legendre nodes in degrees (a CUSTOM latitude spacing)."""
  return np.sort(np.rad2deg(np.arcsin(np.polynomial.legendre.leggauss(n)[0])))


def grid(lon, lat, periodic=True, includes_poles=True):
  return rg.Grid(longitudes=np.asarray(lon), latitudes=np.asarray(lat),
                 periodic=periodic, includes_poles=includes_poles)


@functools.lru_cache(maxsize=None)
def _weights(src, tgt):
  r = rg.ConservativeRegridder(src, tgt)
  return r._weights  # pylint: disable=protected-access


FIELDS = ('z500', 't', 'sp', 'q', 'u', 'v', 'precip', 'sst')


def field(kind, lon_deg, lat_deg, seed):
  """A float32 (nlon, nlat) field of `kind` with realistic magnitudes."""
  rs = np.random.RandomState(seed)
  lo = np.deg2rad(np.asarray(lon_deg, np.float64))[:, None]
  la = np.deg2rad(np.asarray(lat_deg, np.float64))[None, :]
  waves = sum(rs.uniform(0.3, 1) / k * np.cos(k * lo + rs.uniform(0, 2 * np.pi))
              * np.cos(la) ** 2 * np.sin(2 * la + rs.uniform(0, 1))
              for k in range(1, 9))
  noise = rs.standard_normal((lo.size, la.size))
  if kind == 'z500':
    f = 5.6e4 - 4.5e3 * np.sin(la) ** 2 + 1.5e3 * waves + 5 * noise
  elif kind == 't':
    f = 300 - 60 * np.sin(la) ** 2 + 8 * waves + 0.5 * noise
  elif kind == 'sp':
    steps = np.floor(3 * (np.sin(3 * lo) * np.cos(2 * la) + 1)) * 6e3
    f = 1.013e5 - np.maximum(steps - 6e3, 0) + 300 * waves + 50 * noise
  elif kind == 'q':
    f = 2e-2 * np.cos(la) ** 4 * 10 ** (-6 * np.abs(np.sin(la))) * (
        1 + 0.3 * waves) * np.exp(0.1 * noise)
    f = np.maximum(f, 1e-8)
  elif kind in ('u', 'v'):
    f = (15 * np.sin(2 * la) if kind == 'u' else 0) + 12 * waves + 3 * noise
  elif kind == 'precip':
    f = np.maximum(noise + 2 * waves - 1.6, 0) * 2e-3
  elif kind == 'sst':
    f = 302 - 30 * np.sin(la) ** 2 + 2 * waves + 0.2 * noise
    land = (np.sin(2 * lo + 1) * np.cos(3 * la) + 0.6 * np.sin(5 * lo) *
            np.sin(4 * la)) > 0.45
    f = np.where(land | (np.abs(la) > np.deg2rad(80)), np.nan, f)
  else:
    raise ValueError(kind)
  return np.asarray(f, np.float32)


def fields(lon_deg, lat_deg, seed, kinds=FIELDS):
  return np.stack([field(k, lon_deg, lat_deg, seed + i)
                   for i, k in enumerate(kinds)])


# ---- cases ------------------------------------------------------------------
@dataclasses.dataclass
class Case:
  name: str
  lon: object       # CsrSpec
  lat: object       # CsrSpec
  x: np.ndarray     # (nfield, nlon_s, nlat_s) float32
  claim: str
  family: str       # 'realistic' | 'structural' | 'inf' | 'raw'
  zero_exact: bool = False
  value_exact: bool = False  # got == float32(want) bit for bit

  @functools.cached_property
  def ref(self):
    return reference(self.lon, self.lat, self.x)

  @property
  def nfield(self):
    return self.x.shape[0]


# (name, source grid, target grid, claim)
def _pairs():
  L, P = lons, lats
  return [
      ('1440x721-240x121', grid(L(1440), P(721)), grid(L(240), P(121)),
       'TMA G2 DPT3 NTAP7'),
      ('1440x721-360x181', grid(L(1440), P(721)), grid(L(360), P(181)),
       'TMA G2 DPT3 NTAP0'),
      ('1440x721-180x91', grid(L(1440), P(721)), grid(L(180), P(91)),
       'LDG DPT3'),
      ('1440x721-144x73', grid(L(1440), P(721)), grid(L(144), P(73)),
       'LDG DPT3'),
      ('1440x721-64x32', grid(L(1440), P(721)),
       grid(L(64), P(32, False), includes_poles=False), 'LDG DPT3'),
      ('720x361-240x121', grid(L(720), P(361)), grid(L(240), P(121)),
       'TMA G2 DPT2 NTAP0'),
      ('360x181-240x121', grid(L(360), P(181)), grid(L(240), P(121)),
       'TMA G2 DPT1 NTAP0'),
      ('240x121-64x32', grid(L(240), P(121)),
       grid(L(64), P(32, False), includes_poles=False), 'TMA G2 DPT1 NTAP0'),
      ('512x256g-240x121', grid(L(512), gaussian_lats(256)),
       grid(L(240), P(121)), 'TMA G2 DPT1 NTAP0'),
      ('2048x1024g-1440x721', grid(L(2048), gaussian_lats(1024)),
       grid(L(1440), P(721)), 'TMA G2 DPT4 NTAP0'),
      ('2048x1024g-240x121', grid(L(2048), gaussian_lats(1024)),
       grid(L(240), P(121)), 'LDG DPT4'),
      ('240x121-1440x721', grid(L(240), P(121)), grid(L(1440), P(721)),
       'TMA G2 DPT1 NTAP0'),
      ('1440x721-1440x721', grid(L(1440), P(721)), grid(L(1440), P(721)),
       'TMA G2 DPT3 NTAP0'),
      ('360x181c-240x121', grid(L(360, rg.LongitudeScheme.CENTER_AT_ZERO),
                                P(181)), grid(L(240), P(121)),
       'TMA G2 DPT1 NTAP0'),
      # limited area: 0 .. 120 E, not periodic (lon_nan target rows)
      ('480x181lam-240x121', grid(np.arange(480) * 0.25, P(181),
                                  periodic=False), grid(L(240), P(121)),
       'TMA G2 DPT1 NTAP0'),
      # pole-less band 60 S .. 60 N (lat_nan target rows)
      ('360x241band-240x121', grid(L(360), np.linspace(-60, 60, 241),
                                   includes_poles=False),
       grid(L(240), P(121)), 'TMA G2 DPT1 NTAP0'),
      ('360x481-30x91', grid(L(360), P(481)), grid(L(30), P(91)),
       'TMA G4 DPT2 NTAP0'),
      ('360x721-50x91', grid(L(360), P(721)), grid(L(50), P(91)),
       'TMA G4 DPT3 NTAP0'),
      ('360x1024g-80x91', grid(L(360), gaussian_lats(1024)),
       grid(L(80), P(91)), 'TMA G4 DPT4 NTAP0'),
      ('360x181-4x19', grid(L(360), P(181)), grid(L(4), P(19)), 'LDG DPT1'),
      ('720x361-6x37', grid(L(720), P(361)), grid(L(6), P(37)), 'LDG DPT2'),
  ]


def grid_pair(name):
  for n, s, t, _ in _pairs():
    if n == name:
      return s, t
  raise KeyError(name)


def _grid_csr(name):
  s, t = grid_pair(name)
  lon_w, lat_w = _weights(s, t)
  return lon_w, lat_w, s


def _band_rows(n_src, n_tgt, width, rs, start=None):
  """n_tgt rows of `width` consecutive sorted taps with positive weights."""
  rows = []
  for i in range(n_tgt):
    b0 = (i * n_src) // n_tgt if start is None else start(i)
    cols = np.arange(b0, b0 + width) % n_src
    cols = np.sort(cols)
    rows.append((cols, rs.uniform(0.05, 1, width).astype(np.float32)))
  return rows


def _raw_pairs():
  """(name, lon CSR, lat CSR, claim) for what grid pairs do not reach."""
  rs = np.random.RandomState(7)
  out = []
  for nlat_s in (1, 2, 3, 5, 255, 256, 257, 512, 513, 768, 769, 1024):
    lon = raw_csr(16, _band_rows(16, 8, 3, rs))
    lat = raw_csr(nlat_s, _band_rows(nlat_s, max(1, nlat_s // 3),
                                     min(3, nlat_s), rs))
    out.append((f'raw-nlat{nlat_s}', lon, lat,
                f'TMA G2 DPT{-(-nlat_s // 256)} NTAP0'))
  # three runs in every group: taps {0, 2, 4} + 6 k
  lon = raw_csr(48, [(np.array([0, 2, 4]) + 6 * i, rs.uniform(.1, 1, 3))
                     for i in range(8)])
  out.append(('raw-three-runs', lon, raw_csr(300, _band_rows(300, 50, 6, rs)),
              'LDG DPT2'))
  # 65 taps per target: G * maxtap > 128 at G = 2 and 4
  lon = raw_csr(260, _band_rows(260, 8, 65, rs))
  out.append(('raw-65-taps', lon, raw_csr(100, _band_rows(100, 30, 4, rs)),
              'LDG DPT1'))
  # empty target rows that are not flagged NaN: 0 / 0
  rows = _band_rows(32, 8, 4, rs)
  rows[3] = (np.zeros(0, np.int32), np.zeros(0, np.float32))
  lat_rows = _band_rows(200, 20, 3, rs)
  lat_rows[0] = (np.zeros(0, np.int32), np.zeros(0, np.float32))
  out.append(('raw-empty-rows', raw_csr(32, rows), raw_csr(200, lat_rows),
              'TMA G2 DPT1 NTAP0'))
  # G = 4 at DPT 1: two targets of a pair tap 30 disjoint rows each (the
  # pair's run does not fit 55 KB), the next pair taps the same rows
  rows = []
  for i in range(8):
    base = (i // 4) * 60 + (i % 2) * 30
    rows.append((np.arange(base, base + 30), rs.uniform(.1, 1, 30)))
  out.append(('raw-g4-dpt1', raw_csr(120, rows),
              raw_csr(256, _band_rows(256, 64, 5, rs)), 'TMA G4 DPT1 NTAP0'))
  # G = 4 with seven taps at DPT 3: each pair's union has three runs, each
  # quadruple's union one run
  rows = []
  for q in range(4):
    o = 28 * q
    rows += [(o + np.arange(0, 7), None),
             (o + np.array([8, 9, 10, 11, 12, 13, 16]), None),
             (o + np.array([7, 14, 15, 17, 18, 19, 20]), None),
             (o + np.arange(21, 28), None)]
  rows = [(c, rs.uniform(.1, 1, 7)) for c, _ in rows]
  out.append(('raw-g4-seven', raw_csr(112, rows),
              raw_csr(700, _band_rows(700, 100, 8, rs)), 'TMA G4 DPT3 NTAP7'))
  return out


def raw_pair(name):
  for n, lon, lat, _ in _raw_pairs():
    if n == name:
      return lon, lat
  raise KeyError(name)


# one carrier per reachable instance for the structural and inf families
CARRIERS = {
    'TMA G2 DPT1 NTAP0': '240x121-64x32',
    'TMA G2 DPT2 NTAP0': '720x361-240x121',
    'TMA G2 DPT3 NTAP0': '1440x721-360x181',
    'TMA G2 DPT3 NTAP7': '1440x721-240x121',
    'TMA G2 DPT4 NTAP0': '2048x1024g-1440x721',
    'TMA G4 DPT1 NTAP0': 'raw-g4-dpt1',
    'TMA G4 DPT2 NTAP0': '360x481-30x91',
    'TMA G4 DPT3 NTAP0': '360x721-50x91',
    'TMA G4 DPT3 NTAP7': 'raw-g4-seven',
    'TMA G4 DPT4 NTAP0': '360x1024g-80x91',
    'LDG DPT1': 'raw-65-taps',
    'LDG DPT2': 'raw-three-runs',
    'LDG DPT3': '1440x721-64x32',
    'LDG DPT4': '2048x1024g-240x121',
}


def carrier(name):
  """(lon CSR, lat CSR) of a grid pair or raw pair."""
  if name.startswith('raw-'):
    return raw_pair(name)
  lon_w, lat_w, _ = _grid_csr(name)
  return lon_w, lat_w


def _footprint(csr, j):
  """Targets of `csr` that tap source j."""
  return {i for i in range(csr.n_tgt) if j in set(taps(csr, i)[0].tolist())}


def spike_positions(lon, lat, nfield=4):
  """Per field, source cells (b, d) with pairwise disjoint footprints at run
  heads and tails, the periodic seam, the first / last latitude and the last
  DPT slice."""
  nlat_s, nlon_s = lat.n_src, lon.n_src
  dpt = -(-nlat_s // 256)
  ds = sorted({d for d in (0, 1, 2, 3, nlat_s // 2, 256 * (dpt - 1),
                           256 * (dpt - 1) + 1, nlat_s - 3, nlat_s - 2,
                           nlat_s - 1) if 0 <= d < nlat_s})
  bs = {0, 1, nlon_s - 2, nlon_s - 1}
  for g in (2, 4):  # first and last row of every run of some groups
    starts = list(range(0, lon.n_tgt, g))
    for a0 in starts[:6] + starts[-3:]:
      rows = np.unique(lon.col_idx[lon.row_ptr[a0]:
                                   lon.row_ptr[min(lon.n_tgt, a0 + g)]])
      if rows.size:
        breaks = np.nonzero(np.diff(rows) != 1)[0]
        bs.update(rows[np.r_[0, breaks + 1]].tolist())
        bs.update(rows[np.r_[breaks, rows.size - 1]].tolist())
  bs = sorted(b for b in bs if 0 <= b < nlon_s)
  fb = {b: _footprint(lon, b) for b in bs}
  fd = {d: _footprint(lat, d) for d in ds}
  cand = [(b, d) for b in bs for d in ds if fb[b] and fd[d]]
  out = []
  for _ in range(nfield):
    taken, mine = [], []
    for b, d in cand:
      if all(not (fb[b] & fb[b2]) or not (fd[d] & fd[d2]) for b2, d2 in taken):
        taken.append((b, d))
    cand = [c for c in cand if c not in taken] or cand
    out.append(taken)
  return out


def structural_cases(inst):
  name = CARRIERS[inst]
  lon, lat = carrier(name)
  shape = (lon.n_src, lat.n_src)
  cases = []
  z = np.zeros((2,) + shape, np.float32)
  z[1] = -0.0
  cases.append(Case(f'{inst}/zeros', lon, lat, z, inst, 'structural',
                    zero_exact=True, value_exact=True))
  cases.append(Case(f'{inst}/all-nan', lon, lat,
                    np.full((1,) + shape, np.nan, np.float32), inst,
                    'structural', value_exact=True))
  x = np.ones((2,) + shape, np.float32)
  x[0, :: max(1, shape[0] // 5), :] = np.nan
  x[0, -1, :] = np.nan
  x[1, :, :: max(1, shape[1] // 4)] = np.nan
  x[1, :, -1] = np.nan
  x[1, 1:3, :] = np.nan
  cases.append(Case(f'{inst}/nan-rows-cols', lon, lat, x, inst, 'structural',
                    value_exact=True))
  pos = spike_positions(lon, lat)
  x = np.zeros((len(pos),) + shape, np.float32)
  for f, cells in enumerate(pos):
    for b, d in cells:
      x[f, b, d] = 1.0
  cases.append(Case(f'{inst}/spikes', lon, lat, x, inst, 'structural',
                    zero_exact=True))
  return cases


def inf_case(inst):
  """+inf, -inf, both signs in one footprint and inf next to NaN, on a
  smooth finite background."""
  name = CARRIERS[inst]
  lon, lat = carrier(name)
  nb, nd = lon.n_src, lat.n_src
  x = np.zeros((4, nb, nd), np.float32)
  x += (1 + 0.5 * np.sin(np.arange(nb) / 7.0))[:, None].astype(np.float32)
  d_last = nd - 1
  x[0, nb // 3, nd // 2] = np.inf
  x[0, 0, 0] = np.inf
  x[1, nb // 2, d_last] = -np.inf
  x[1, nb - 1, nd // 3] = -np.inf
  x[2, nb // 4, nd // 2] = np.inf
  x[2, min(nb - 1, nb // 4 + 1), nd // 2] = -np.inf
  x[3, nb // 5, nd // 4] = np.inf
  x[3, min(nb - 1, nb // 5 + 1), nd // 4] = np.nan
  x[3, nb // 5, min(nd - 1, nd // 4 + 1)] = np.nan
  return Case(f'{inst}/inf', lon, lat, x, inst, 'inf')


def realistic_cases():
  out = []
  for i, (name, s, t, claim) in enumerate(_pairs()):
    lon_w, lat_w = _weights(s, t)
    x = fields(s.longitudes, s.latitudes, 100 * i)
    out.append(Case(name, lon_w, lat_w, x, claim, 'realistic'))
  return out


def raw_cases():
  out = []
  for i, (name, lon, lat, claim) in enumerate(_raw_pairs()):
    rs = np.random.RandomState(1000 + i)
    x = (5e4 + 300 * rs.standard_normal((3, lon.n_src, lat.n_src))).astype(
        np.float32)
    x[1] = rs.standard_normal(x[1].shape)
    x[2][rs.rand(*x[2].shape) < 0.1] = np.nan
    out.append(Case(name, lon, lat, x, claim, 'raw'))
  return out


@functools.lru_cache(maxsize=None)
def all_cases():
  cases = realistic_cases() + raw_cases()
  for inst in INSTANCES:
    cases += structural_cases(inst)
    cases.append(inf_case(inst))
  return tuple(cases)


def case_names():
  """Names without building the fields (for parametrisation)."""
  names = [n for n, *_ in _pairs()] + [n for n, *_ in _raw_pairs()]
  for inst in INSTANCES:
    names += [f'{inst}/{k}' for k in ('zeros', 'all-nan', 'nan-rows-cols',
                                      'spikes', 'inf')]
  return names


def get_case(name):
  for c in all_cases():
    if c.name == name:
      return c
  raise KeyError(name)


def bad_csr_pairs():
  """(name, lon CSR, lat CSR) that wb2_regrid_conservative must reject."""
  rs = np.random.RandomState(3)
  good = _band_rows(16, 8, 3, rs)
  lat = raw_csr(40, _band_rows(40, 10, 4, rs))
  unsorted = list(good)
  c, v = unsorted[2]
  unsorted[2] = (c[::-1].copy(), v)
  dup = list(good)
  c, v = dup[5]
  dup[5] = (np.array([c[0], c[0], c[1]]), v)
  lat_dup = _band_rows(40, 10, 4, rs)
  c, v = lat_dup[4]
  lat_dup[4] = (np.array([c[0], c[1], c[1], c[3]]), v)
  return [('lon-unsorted', raw_csr(16, unsorted), lat),
          ('lon-duplicate', raw_csr(16, dup), lat),
          ('lat-duplicate', raw_csr(16, good), raw_csr(40, lat_dup))]

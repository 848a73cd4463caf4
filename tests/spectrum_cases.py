"""Seeded zonal-spectrum cases with float64 answers and a per-bin error bound
(K4: csrc/spectrum_pfa.cu, csrc/spectrum.cu).

Two families:
  * realistic rows, built from a prescribed amplitude spectrum with seeded
    phases and rounded to float32: z500-like (5.5e4 + k^-3, with and without a
    Gaussian taper at k ~ 300), temperature (220-310 K with a latitude
    gradient), surface pressure (~1e5), specific humidity (1e-8 .. 1e-2), a
    wind component with a negative mean, and white noise with and without an
    offset;
  * structural rows with exact answers: constant, zeros, +-0, a single spike,
    alternating +-1 (Nyquist only), pure tones at chosen bins, and a single NaN
    or +-inf placed in row A / row B of a pair, the first / last pair of a
    G-group and the last row of an odd nrow (the row the padding repeats).

The target is the exact DFT of the float32 input: the oracle's float64 rfft.

Per-bin bound (DESIGN K4).  u = 2^-24, D = max_n |x_n - mean|, F_k the
forward-normalised DFT of the float32 row, c_k = 1 for k = 0 and 2 otherwise,
sigma the row's scale:
    e        = C_plan u D
    |got_k - want_k| <= c_k sigma (2 |F_k| e + e^2) + m u want_k
C_plan = 2 L / sqrt(N / 2) for N > 2 (2 L for N = 2), L the number of
rounding levels on the path from an input to a bin (the shift, every radix's
butterfly levels, the inter-stage twiddles, the split).  The factor 2 covers
|x_n - s| <= 2 D for any shift s that is one of the row's values or its mean;
1 / sqrt(N / 2) is the random-walk growth of the N / 2 independent roundings
that reach one bin, against the worst case in which they all align.  Bin 0
adds 4 u max|x| to e (N s is added back there).  m = 6 covers the power FMA,
the float32 scale and the final product; a same-sign float32 sum of n terms
adds n - 1."""
import numpy as np

U = 2.0 ** -24
NSM = 132  # H100 SXM
R_EARTH = 1000 * (6357 + 6378) / 2

# the prime-factor plans of spectrum_pfa.cu: N -> (RA, RB, RC, G, MINB)
PFA_PLANS = {1440: (9, 16, 5, 2, 3), 720: (9, 8, 5, 5, 2), 240: (3, 8, 5, 6, 2)}
# the fixed Stockham plans of spectrum.cu: N2 -> radices
FIXED_PLANS = {720: (16, 9, 5), 360: (9, 8, 5), 180: (9, 5, 4), 120: (8, 5, 3),
               256: (16, 16), 32: (16, 2)}
_LEVELS = {1: 0, 2: 1, 3: 2, 4: 2, 5: 3, 8: 5, 9: 6, 16: 6}


def factorize(n2):
  """spectrum.cu factorize(): greedy 16, 9, 8, 5, 4, 3, 2."""
  out = []
  for r in (16, 9, 8, 5, 4, 3, 2):
    while n2 % r == 0:
      out.append(r)
      n2 //= r
  assert n2 == 1
  return out or [1]


def path_for(n, aligned=True, force=None):
  """The path wb2_zonal_spectrum takes: 'pfa', 'fixed' or 'generic'."""
  if force in (None, 'pfa') and aligned and n in PFA_PLANS:
    return 'pfa'
  if force != 'generic' and n // 2 in FIXED_PLANS:
    return 'fixed'
  return 'generic'


def levels(n, path):
  """L: rounding levels from an input to a bin on `path`."""
  if path == 'pfa':
    ra, rb, rc = PFA_PLANS[n][:3]
    return 1 + _LEVELS[ra] + _LEVELS[rb] + _LEVELS[rc] + 4
  radices = FIXED_PLANS[n // 2] if path == 'fixed' else factorize(n // 2)
  return 1 + sum(_LEVELS[r] for r in radices) + 2 * (len(radices) - 1) + 4


def c_plan(n, path):
  lv = levels(n, path)
  return 2.0 * lv if n <= 2 else 2.0 * lv / np.sqrt(n / 2)


def want(x, scale):
  """[..., row, k] float64: |rfft(norm=forward)|^2 c_k scale[row]."""
  f = np.fft.rfft(np.asarray(x, np.float64), axis=-1, norm='forward')
  s = (f * np.conj(f)).real
  s[..., 1:] *= 2
  return s * np.asarray(scale, np.float64)[:, None]


def bound(x, scale, path, nacc=1):
  """Per-bin bound of |got - want| for every row of x ([..., row, N]); with
  nacc > 1 the rows of x[i] are summed over the leading axis (time)."""
  xd = np.asarray(x, np.float64)
  n = xd.shape[-1]
  d = np.max(np.abs(xd - xd.mean(-1, keepdims=True)), axis=-1, keepdims=True)
  f = np.abs(np.fft.rfft(xd, axis=-1, norm='forward'))
  e = c_plan(n, path) * U * d * np.ones_like(f)
  e[..., 0] += 4 * U * np.max(np.abs(xd), axis=-1)
  ck = np.full(f.shape[-1], 2.0)
  ck[0] = 1.0
  sc = np.abs(np.asarray(scale, np.float64))[:, None]
  w = want(xd, scale)
  b = ck * sc * (2 * f * e + e * e) + 6 * U * np.abs(w)
  return b, w


# ---- rows ---------------------------------------------------------------------
def synth(n, rs, slope, std, taper=None):
  """Zero-mean float64 row with power ~ k^-slope, random phases, scaled to
  `std`; `taper`: Gaussian roll-off of the amplitude past that wavenumber."""
  k = np.arange(n // 2 + 1, dtype=np.float64)
  amp = np.zeros_like(k)
  amp[1:] = k[1:] ** (-slope / 2)
  if taper is not None:
    amp[1:] *= np.exp(-np.maximum(k[1:] - taper, 0) ** 2 / (2 * (taper / 10) ** 2))
  ph = rs.uniform(0, 2 * np.pi, k.size)
  spec = amp * np.exp(1j * ph)
  spec[-1] = spec[-1].real
  row = np.fft.irfft(spec, n)
  return row * (std / row.std())


def realistic(kind, nrow, n, seed):
  """[nrow, n] float32 rows of one realistic family."""
  rs = np.random.RandomState(seed)
  rows = []
  for r in range(nrow):
    frac = r / max(nrow - 1, 1)
    if kind == 'z500':
      v = 5.5e4 + synth(n, rs, 3, 1500)
    elif kind == 'z500_tapered':
      v = 5.5e4 + synth(n, rs, 3, 1500, taper=min(300, n // 5))
    elif kind == 'temperature':
      v = 220 + 90 * np.sin(np.pi * frac) + synth(n, rs, 3, 8)
    elif kind == 'pressure':
      v = 1e5 + synth(n, rs, 3, 1000, taper=min(300, n // 5))
    elif kind == 'humidity':
      m = 10 ** (-8 + 6 * frac)
      v = m * (1 + 0.4 * synth(n, rs, 2, 1) / 3)
    elif kind == 'wind':
      v = -5 + synth(n, rs, 5 / 3, 10)
    elif kind == 'white':
      v = rs.standard_normal(n)
    elif kind == 'white_offset':
      v = 3 + rs.standard_normal(n)
    else:
      raise ValueError(kind)
    rows.append(v)
  return np.asarray(rows).astype(np.float32)


REALISTIC = ('z500', 'z500_tapered', 'temperature', 'pressure', 'humidity',
             'wind', 'white', 'white_offset')
# the families whose mean is large against their variation
LARGE_MEAN = ('z500', 'z500_tapered', 'temperature', 'pressure')


def crt_bins(n):
  """Good-Thomas output map of the PFA plan for N = n: bin p of X lives at
  (kA, kB, kC) = (p mod RA, p mod RB, p mod RC) of the N2-point transform."""
  ra, rb, rc = PFA_PLANS[n][:3]
  return ra, rb, rc


def tone_bins(n):
  """Bins p for pure tones: 1, N/2 - 1, the Nyquist bin and, for PFA sizes,
  one bin of every residue class (p mod RA, p mod RB) of the stage-C tasks
  and of every residue class mod RC."""
  n2 = n // 2
  bins = {1, max(n2 - 1, 1), n2}
  if n in PFA_PLANS:
    ra, rb, rc = crt_bins(n)
    need = {(a, b) for a in range(ra) for b in range(rb)}
    needc = set(range(rc))
    for p in range(1, n2 + 1):  # p = 0 is a constant row, not a tone
      key = (p % ra, p % rb)
      if key in need or p % rc in needc:
        bins.add(p)
        need.discard(key)
        needc.discard(p % rc)
  return sorted(bins)


def tone(n, p, amp=1.0, phase=0.3):
  t = np.arange(n)
  return (amp * np.cos(2 * np.pi * p * t / n + phase)).astype(np.float32)


def structural(n):
  """(name, row, exact power of the forward-normalised DFT or None)."""
  out = []
  k = n // 2 + 1
  z = np.zeros(k)
  c = np.full(n, 287.5, np.float32)
  e = z.copy()
  e[0] = 287.5 ** 2
  out.append(('constant', c, e))
  out.append(('zeros', np.zeros(n, np.float32), z.copy()))
  pm = np.zeros(n, np.float32)
  pm[1::2] = -0.0
  out.append(('signed_zeros', pm, z.copy()))
  sp = np.zeros(n, np.float32)
  sp[3 % n] = 2.0
  e = np.full(k, 2 * (2.0 / n) ** 2)
  e[0] = (2.0 / n) ** 2
  if n % 2 == 0:
    e[-1] = 2 * (2.0 / n) ** 2
  out.append(('spike', sp, e))
  alt = np.where(np.arange(n) % 2 == 0, 1.0, -1.0).astype(np.float32)
  e = z.copy()
  e[-1] = 2.0  # the Nyquist bin is doubled as in the reference (:600)
  out.append(('alternating', alt, e))
  return out


def pfa_geometry(n, nrow, nslot=1, ntime=1):
  """(npair, ngroup, nchunk of mode 2) that pfa::launch computes on NSM SMs."""
  g, minb = PFA_PLANS[n][3], PFA_PLANS[n][4]
  npair = (nrow + 1) // 2
  ngroup = (npair + g - 1) // g
  want_jobs = NSM * minb * 4
  nchunk = max(1, (want_jobs + nslot - 1) // nslot)
  nchunk = min(nchunk, ngroup)
  gpc = (ngroup + nchunk - 1) // nchunk
  return npair, ngroup, (ngroup + gpc - 1) // gpc


def nonfinite_rows(n):
  """Row indices that put a NaN / inf in row A and row B of a pair, the first
  and last pair of a G-group and the last row of an odd nrow, for the PFA
  plan of N = n: returns (nrow, {label: row})."""
  g = PFA_PLANS[n][3]
  nrow = 2 * (2 * g) + 3  # two whole groups, then a partial one ending on an odd row
  return nrow, {'row_a': 0, 'row_b': 1, 'first_pair_of_group': 2 * g,
                'last_pair_of_group': 2 * g + 2 * (g - 1) + 1,
                'last_odd_row': nrow - 1}


# ---- float32 model of the PFA plan -------------------------------------------
def _dft_f32(v, axis):
  """Float32 DFT along `axis` of a complex64 array, twiddles rounded once from
  float64, sums in float32 in index order."""
  r = v.shape[axis]
  idx = np.arange(r)
  w = np.exp(-2j * np.pi * np.outer(idx, idx) / r).astype(np.complex64)
  vm = np.moveaxis(v, axis, -1)
  out = np.zeros_like(vm)
  for j in range(r):
    out = out + vm[..., j:j + 1] * w[:, j]
  return np.moveaxis(out.astype(np.complex64), -1, axis)


def pfa_model(x, shift):
  """Power spectrum |X_k|^2 c_k / N^2 of float32 rows x [rows, N] through the
  prime-factor plan in float32: Good's input map, three radix DFTs, the
  real-input split with float32 twiddles from the same double table as
  build_tables, the power in float32.  shift=True transforms x - x[0] and adds
  N x[0] back into bin 0."""
  x = np.asarray(x, np.float32)
  n = x.shape[-1]
  ra, rb, rc = PFA_PLANS[n][:3]
  n2 = n // 2
  s = x[:, :1] if shift else np.zeros_like(x[:, :1])
  y = (x - s).astype(np.float32)
  zc = (y[:, 0::2] + np.complex64(1j) * y[:, 1::2]).astype(np.complex64)
  sa, sb, sc = n2 // ra, n2 // rb, n2 // rc
  na, nb, nc = np.meshgrid(np.arange(ra), np.arange(rb), np.arange(rc), indexing='ij')
  work = zc[:, (sa * na + sb * nb + sc * nc) % n2]  # [rows, RA, RB, RC]
  for ax in (1, 2, 3):
    work = _dft_f32(work, ax)
  ea = _idem(n2, ra)
  eb = _idem(n2, rb)
  ec = _idem(n2, rc)
  z = np.zeros_like(zc)
  z[:, (ea * na + eb * nb + ec * nc) % n2] = work
  p = np.arange(n2 + 1)
  zp = z[:, p % n2]
  zq = np.conj(z[:, (n2 - p) % n2])
  e = (zp + zq).astype(np.complex64)
  d = (zp - zq).astype(np.complex64)
  w = np.exp(-2j * np.pi * p / n).astype(np.complex64)
  xk = (e + (w * (np.complex64(-1j) * d)).astype(np.complex64)).astype(np.complex64)
  xk[:, 0] = xk[:, 0] + np.float32(2 * n) * s[:, 0]
  pw = (xk.real * xk.real + xk.imag * xk.imag).astype(np.float32)
  ck = np.full(n2 + 1, 2.0, np.float32)
  ck[0] = 1.0
  return pw.astype(np.float64) * ck / (4.0 * n * n)


def _idem(n2, r):
  m = n2 // r
  v = m
  while v % r != 1 % r:
    v += m
  return v % n2

"""ctypes binding of libwb2b200.so (the C ABI in include/wb2b200.h).

There is NO CPU fallback: if the shared library is missing, or no H100 is
visible when a context is created, the calls raise `Wb2Error`.
"""
from __future__ import annotations

import ctypes as C
import os
import threading
from typing import Optional

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libwb2b200.so')

F32, F64 = 0, 1
MAX_REGIONS = 32
DET_NSTAT = 10
ENS_NSTAT = 10
MAP_BIAS, MAP_MSE, MAP_MAE = 0, 1, 2
# bits of wb2_ens_maps' stat_mask
ENS_SKILL, ENS_SPREAD, ENS_MEAN_SE, ENS_VARIANCE, ENS_DEBIASED = 1, 2, 4, 8, 16
ENS_CRPS = 32


class Wb2Error(RuntimeError):
  """Raised when the native library reports an error (or is missing)."""


class Weights(C.Structure):
  """struct wb2_weights (include/wb2b200.h)."""
  _fields_ = [
      ('nrow', C.c_int32),
      ('ncol', C.c_int32),
      ('row_stride', C.c_int64),
      ('nregion', C.c_int32),
      ('nseg', C.c_int32),
      ('row_w', C.POINTER(C.c_double)),
      ('seg_start', C.POINTER(C.c_int32)),
      ('seg_w', C.POINTER(C.c_double)),
      ('col_w', C.POINTER(C.c_float)),
      ('cell_w', C.c_void_p),
      ('zero_skip', C.c_int32),
  ]


class Csr(C.Structure):
  """struct wb2_csr (include/wb2b200.h)."""
  _fields_ = [
      ('n_src', C.c_int32),
      ('n_tgt', C.c_int32),
      ('row_ptr', C.POINTER(C.c_int32)),
      ('col_idx', C.POINTER(C.c_int32)),
      ('val', C.POINTER(C.c_float)),
      ('nan_row', C.POINTER(C.c_uint8)),
  ]


_lib = None
_lib_lock = threading.Lock()

_P = C.c_void_p
_I64P = C.POINTER(C.c_int64)
_I32P = C.POINTER(C.c_int32)

# name -> (restype, argtypes); every symbol include/wb2b200.h declares
PROTOTYPES = {
    'wb2_version': (C.c_int, []),
    'wb2_last_error': (C.c_char_p, []),
    'wb2_has_cuda': (C.c_int, []),
    'wb2_launch_count': (C.c_int64, [_P]),
    'wb2_create': (C.c_int, [C.c_int, C.POINTER(_P)]),
    'wb2_destroy': (C.c_int, [_P]),
    'wb2_set_stream': (C.c_int, [_P, _P]),
    'wb2_get_stream': (_P, [_P]),
    'wb2_synchronize': (C.c_int, [_P]),
    'wb2_wait_stream': (C.c_int, [_P, _P]),
    'wb2_stream_wait': (C.c_int, [_P, _P]),
    'wb2_malloc': (C.c_int, [_P, C.c_size_t, C.POINTER(_P)]),
    'wb2_free': (C.c_int, [_P, _P]),
    'wb2_host_alloc': (C.c_int, [_P, C.c_size_t, C.POINTER(_P)]),
    'wb2_host_free': (C.c_int, [_P, _P]),
    'wb2_memcpy_h2d': (C.c_int, [_P, _P, _P, C.c_size_t]),
    'wb2_memcpy_d2h': (C.c_int, [_P, _P, _P, C.c_size_t]),
    'wb2_memset': (C.c_int, [_P, _P, C.c_int, C.c_size_t]),
    'wb2_det_metrics': (C.c_int, [_P, _P, _P, _P, C.c_int, C.c_int64, _I64P,
                                  _I64P, _I64P, C.POINTER(Weights), C.c_int,
                                  _P]),
    'wb2_det_metrics_vector': (C.c_int, [_P, _P, _P, _P, _P, C.c_int,
                                         C.c_int64, _I64P, _I64P, _I64P, _I64P,
                                         C.POINTER(Weights), C.c_int, _P]),
    'wb2_det_metrics_host': (C.c_int, [_P, _P, _P, _P, C.c_int, C.c_int64,
                                       _I64P, _I64P, _I64P, C.POINTER(Weights),
                                       C.c_int, _P]),
    'wb2_ens_metrics': (C.c_int, [_P, _P, _P, C.c_int, C.c_int32, C.c_int64,
                                  C.c_int64, _I64P, _I64P, C.POINTER(Weights),
                                  C.c_int, _P]),
    'wb2_energy_score': (C.c_int, [_P, _P, _P, C.c_int, C.c_int32, C.c_int64,
                                   C.c_int64, _I64P, _I64P, C.POINTER(Weights),
                                   _P]),
    'wb2_det_maps': (C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_int64,
                               C.c_int32, _I64P, _I64P, C.c_int32, C.c_int32,
                               C.c_int64, C.c_int, _P]),
    'wb2_ens_maps': (C.c_int, [_P, _P, _P, C.c_int, C.c_int32, C.c_int64,
                               C.c_int64, C.c_int32, _I64P, _I64P, C.c_int32,
                               C.c_int32, C.c_int64, C.c_int32, C.c_int, _P]),
    'wb2_ens_threshold_metrics': (C.c_int, [
        _P, _P, _P, C.c_int, C.c_int32, C.c_int64, C.c_int64, _I64P, _I64P,
        C.c_int32, _P, _I64P, _P, _I64P, C.POINTER(C.c_double),
        C.POINTER(Weights), C.c_int, _P]),
    'wb2_ens_threshold_maps': (C.c_int, [
        _P, _P, _P, C.c_int, C.c_int32, C.c_int64, C.c_int64, C.c_int32, _I64P,
        _I64P, C.c_int32, _P, _I64P, _P, _I64P, C.POINTER(C.c_double),
        C.c_int32, C.c_int32, C.c_int64, C.c_int32, C.c_int, _P]),
    'wb2_gaussian_metrics': (C.c_int, [
        _P, _P, _P, _P, C.c_int, C.c_int64, _I64P, _I64P, _I64P, C.c_int32,
        _P, _I64P, _P, _I64P, C.POINTER(C.c_double), C.POINTER(Weights),
        C.c_int, _P]),
    'wb2_regrid_conservative': (C.c_int, [_P, _P, _P, C.c_int64, C.c_int64,
                                          C.c_int64, C.POINTER(Csr),
                                          C.POINTER(Csr)]),
    'wb2_wind_speed': (C.c_int, [_P, _P, _P, _P, C.c_int64]),
    'wb2_wind_dynamics': (C.c_int, [
        _P, C.c_int, _P, _P, _P, C.c_int64, C.c_int32, C.c_int32, C.c_int32,
        C.c_int64, C.c_int64, C.POINTER(C.c_double), C.c_int,
        C.POINTER(C.c_double), C.c_int, C.POINTER(C.c_double),
        C.POINTER(C.c_double), C.POINTER(C.c_double), _P]),
    'wb2_column_integral': (C.c_int, [
        _P, C.c_int, C.c_int, _P, _P, _P, C.c_int64, C.c_int64, C.c_int32,
        C.c_int64, C.c_int32, C.c_int64, C.POINTER(C.c_double), _P]),
    'wb2_lapse_rate': (C.c_int, [
        _P, C.c_int, _P, _P, C.c_int64, C.c_int32, C.c_int64,
        C.POINTER(C.c_double), C.c_int, _P]),
    'wb2_relative_humidity': (C.c_int, [
        _P, C.c_int, C.c_int, _P, _P, C.c_int64, C.c_int32, C.c_int64,
        C.POINTER(C.c_double), _P]),
    'wb2_ens_mean': (C.c_int, [_P, _P, C.c_int32, C.c_int64, C.c_int64, _I64P,
                               C.c_int64, C.c_int, _P]),
    'wb2_spectrum_interp': (C.c_int, [_P, _P, C.c_int64, C.c_int32, C.c_int32,
                                      C.POINTER(C.c_double), C.c_int32,
                                      C.POINTER(C.c_double), _P]),
    'wb2_rank_histogram': (C.c_int, [
        _P, _P, _P, C.c_int32, C.c_int64, C.c_int64, C.c_int32, _I64P, _I64P,
        C.c_int32, C.c_int32, C.c_int64, C.c_int32, C.c_int32, C.c_uint64,
        _P]),
    'wb2_seeps_maps': (C.c_int, [
        _P, _P, C.c_int, _P, C.c_int, _P, C.c_int, _P, C.c_int, C.c_int64,
        C.c_int32, _I64P, _I64P, _I64P, _I64P, C.c_int32, C.c_int32,
        C.c_int64, C.c_int64, C.c_double, C.c_double, C.c_double, C.c_int,
        _P]),
    'wb2_regrid_gather': (C.c_int, [_P, _P, _P, C.c_int64, C.c_int64, C.c_int64,
                                    C.c_int32, C.c_int32,
                                    C.POINTER(C.c_int32)]),
    'wb2_regrid_bilinear': (C.c_int, [
        _P, _P, _P, C.c_int64, C.c_int64, C.c_int64, C.c_int32, C.c_int32,
        C.c_int32, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32),
        C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_int32),
        C.POINTER(C.c_float)]),
    'wb2_zonal_spectrum': (C.c_int, [_P, _P, C.c_int64, C.c_int32, C.c_int32,
                                     C.POINTER(C.c_double), _P, C.c_int32,
                                     C.c_int64]),
    'wb2_zonal_spectrum_latsum': (C.c_int, [_P, _P, C.c_int64, C.c_int32,
                                            C.c_int32, C.POINTER(C.c_double),
                                            _P, C.c_int64]),
    'wb2_set_slab_cache': (C.c_int, [_P, C.c_size_t]),
    'wb2_transfer_stats': (C.c_int64, [_P, C.c_int]),
    'wb2_reset_transfer_stats': (C.c_int, [_P]),
    'wb2_ens_metrics_host': (C.c_int, [_P, _P, _P, C.c_int, C.c_int32,
                                       C.c_int64, C.c_int64, _I64P, _I64P,
                                       C.POINTER(Weights), C.c_int, _P]),
    'wb2_regrid_conservative_host': (C.c_int, [_P, _P, _P, C.c_int64,
                                               C.c_int64, C.c_int64,
                                               C.POINTER(Csr),
                                               C.POINTER(Csr)]),
    'wb2_zonal_spectrum_host': (C.c_int, [_P, _P, C.c_int64, C.c_int32,
                                          C.c_int32, C.POINTER(C.c_double), _P,
                                          C.c_int32, C.c_int64]),
    'wb2_zonal_spectrum_latsum_host': (C.c_int, [_P, _P, C.c_int64, C.c_int32,
                                                 C.c_int32,
                                                 C.POINTER(C.c_double), _P,
                                                 C.c_int64]),
    'wb2_climatology': (C.c_int, [
        _P, _P, C.c_int, C.c_int64, C.c_int64, C.c_int64, _I64P, _I32P,
        C.c_int32, C.c_int32, C.c_int32, _I64P, _I64P, _I32P, _I32P, C.c_int32,
        C.c_int32, C.c_int32, _P, _P]),
    'wb2_climatology_host': (C.c_int, [
        _P, _P, C.c_int, C.c_int64, C.c_int64, C.c_int64, _I64P, _I32P,
        C.c_int32, C.c_int32, C.c_int32, _I64P, _I64P, _I32P, _I32P, C.c_int32,
        C.c_int32, C.c_int32, C.c_size_t, _P, _P]),
    'wb2_climatology_quantile': (C.c_int, [
        _P, _P, C.c_int, C.c_int64, C.c_int64, C.c_int64, _I64P, _I32P,
        C.c_int32, C.c_int32, C.c_int32, _I64P, _I64P, _I32P, _I32P, C.c_int32,
        C.c_int32, C.c_int32, C.POINTER(C.c_double), C.c_int32, C.c_double, _P,
        _P]),
    'wb2_climatology_quantile_host': (C.c_int, [
        _P, _P, C.c_int, C.c_int64, C.c_int64, C.c_int64, _I64P, _I32P,
        C.c_int32, C.c_int32, C.c_int32, _I64P, _I64P, _I32P, _I32P, C.c_int32,
        C.c_int32, C.c_int32, C.POINTER(C.c_double), C.c_int32, C.c_double,
        C.c_size_t, _P, _P]),
    'wb2_time_window_stats': (C.c_int, [
        _P, _P, C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_int64, _I64P,
        _I32P, C.c_int32, C.c_int, _P, _P, _P, _P]),
    'wb2_time_window_stats_host': (C.c_int, [
        _P, _P, C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_int64, _I64P,
        _I32P, C.c_int32, C.c_int, C.c_size_t, _P, _P, _P, _P]),
    'wb2_precip_accumulation': (C.c_int, [
        _P, _P, C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_int32, C.c_int,
        _P]),
    'wb2_precip_accumulation_host': (C.c_int, [
        _P, _P, C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_int32, C.c_int,
        C.c_size_t, _P]),
    'wb2_quantile': (C.c_int, [
        _P, _P, C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_int32,
        C.POINTER(C.c_double), C.c_int, _P]),
    'wb2_quantile_host': (C.c_int, [
        _P, _P, C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_int32,
        C.POINTER(C.c_double), C.c_int, C.c_size_t, _P]),
    'wb2_average': (C.c_int, [
        _P, _P, C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_int64,
        C.c_int64, C.POINTER(C.c_double), C.c_int64, C.c_int64, C.c_int, _P,
        _P, _P]),
    'wb2_average_host': (C.c_int, [
        _P, _P, C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_int64,
        C.c_int64, C.POINTER(C.c_double), C.c_int64, C.c_int64, C.c_int,
        C.c_size_t, _P, _P, _P]),
    'wb2_slab_gather': (C.c_int, [
        _P, _P, C.c_int, C.c_int64, C.c_int64, C.c_int64, _I64P, _P, C.c_int]),
    'wb2_slab_gather_host': (C.c_int, [
        _P, _P, C.c_int, C.c_int64, C.c_int64, C.c_int64, _I64P, C.c_size_t, _P,
        C.c_int]),
}
# wb2_average: samples per chunk of the fixed summation order
AVERAGE_CHUNK = 65536
# wb2_quantile: quantiles per call
MAX_QUANTILES = 128
# wb2_climatology_quantile: quantiles per call, nitem * window_size per window
CLIM_MAX_QUANTILES = 16
CLIM_QUANTILE_MAX_SAMPLES = 8192


def load_library():
  """Loads libwb2b200.so (once).  Raises Wb2Error if it has not been built."""
  global _lib
  with _lib_lock:
    if _lib is not None:
      return _lib
    if not os.path.exists(LIB_PATH):
      raise Wb2Error(
          f'{LIB_PATH} not found: build it with '
          '`python -c "import __graft_entry__ as g; g.build()"` or '
          '`make -C weatherbench2_b200/csrc`.  There is no CPU fallback.')
    lib = C.CDLL(LIB_PATH)
    for name, (restype, argtypes) in PROTOTYPES.items():
      fn = getattr(lib, name)  # AttributeError if the ABI is incomplete
      fn.restype = restype
      fn.argtypes = argtypes
    _lib = lib
    return lib


def check(rc: int):
  if rc != 0:
    msg = load_library().wb2_last_error()
    raise Wb2Error(f'libwb2b200 error {rc}: {msg.decode() if msg else "?"}')


def _as_ptr(a: Optional[np.ndarray], ctype):
  if a is None:
    return None
  return a.ctypes.data_as(C.POINTER(ctype))


# entry points that enqueue kernels (or staged copies) on the context's stream
_COMPUTE = frozenset(n for n in PROTOTYPES if n not in (
    'wb2_version', 'wb2_last_error', 'wb2_has_cuda', 'wb2_launch_count',
    'wb2_create', 'wb2_destroy', 'wb2_set_stream', 'wb2_get_stream',
    'wb2_synchronize', 'wb2_wait_stream', 'wb2_stream_wait', 'wb2_malloc',
    'wb2_free', 'wb2_host_alloc', 'wb2_host_free', 'wb2_set_slab_cache',
    'wb2_transfer_stats', 'wb2_reset_transfer_stats'))


def _torch_current_stream(device: int):
  """cudaStream_t of torch's current stream on `device`, or None when torch
  has not been imported / has no CUDA context (nothing to order against)."""
  import sys  # pylint: disable=import-outside-toplevel
  torch = sys.modules.get('torch')
  if torch is None:
    return None
  try:
    if not (torch.cuda.is_available() and torch.cuda.is_initialized()):
      return None
    return int(torch.cuda.current_stream(device).cuda_stream)
  except Exception:  # pylint: disable=broad-except
    return None


class _LockedLib:
  """The library with every call into it serialised by the context's lock.  A
  wb2_ctx (stream, descriptor slots, scratch) is not re-entrant, ctypes drops
  the GIL during a call, and the reference's callers may evaluate chunks from
  several threads (Beam DirectRunner, weatherbench2/evaluation.py:697, 733)
  against the process-wide default context.  Error strings are thread-local
  on the C side, so `check()` may read them after the lock is released.

  Stream ordering: the context's stream is non-blocking, so nothing orders it
  implicitly against torch's streams.  Every compute entry point is therefore
  bracketed by wb2_wait_stream / wb2_stream_wait on torch's CURRENT stream
  (device-side event waits, no host blocking): kernels see inputs that torch
  is still producing, and torch consumers / `.cpu()` see finished outputs.
  Both are no-ops when the context shares torch's stream (bench.py)."""

  def __init__(self, lib, lock, owner=None):
    self._lib = lib
    self._lock = lock
    self._owner = owner

  def __getattr__(self, name):
    fn = getattr(self._lib, name)
    lock = self._lock
    if name in _COMPUTE and self._owner is not None:
      owner, raw = self._owner, self._lib

      def call(*args):
        with lock:
          s = _torch_current_stream(owner.device)
          if s is None:
            return fn(*args)
          rc = raw.wb2_wait_stream(owner.handle, _P(s))
          if rc != 0:
            return rc
          rc = fn(*args)
          rc2 = raw.wb2_stream_wait(owner.handle, _P(s))
          return rc if rc != 0 else rc2
    else:

      def call(*args):
        with lock:
          return fn(*args)

    call.__name__ = name
    setattr(self, name, call)  # cache: __getattr__ only runs on a miss
    return call


class Context:
  """A wb2_ctx: one CUDA device + stream + descriptor arenas.  Safe to share
  between threads (calls are serialised per context)."""

  def __init__(self, device: int = 0):
    self._lock = threading.RLock()
    self.device = int(device)
    self.lib = _LockedLib(load_library(), self._lock, self)
    h = _P()
    check(self.lib.wb2_create(int(device), C.byref(h)))
    self.handle = h
    self._slab_cache_bytes = 0
    self._pinned_pool: dict = {}
    self._pinned_pool_limit = int(os.environ.get('WB2_PINNED_POOL_MB',
                                                 '4096')) << 20
    self._closed = False

  def close(self):
    if not self._closed:
      for bufs in self._pinned_pool.values():  # pooled result buffers
        for ptr in bufs:
          try:
            self.lib.wb2_host_free(self.handle, _P(ptr))
          except Exception:  # pylint: disable=broad-except
            pass
      self._pinned_pool.clear()
      # device copies of LandRegion masks (_spatial.build_weights)
      for ptr in self.__dict__.pop('_cell_weight_cache', {}).values():
        try:
          self.lib.wb2_free(self.handle, _P(ptr))
        except Exception:  # pylint: disable=broad-except
          pass
      self._closed = True
      self.lib.wb2_destroy(self.handle)

  def __del__(self):
    try:
      self.close()
    except Exception:  # pylint: disable=broad-except
      pass

  # -- streams / memory -------------------------------------------------------
  def set_stream(self, cuda_stream: int):
    check(self.lib.wb2_set_stream(self.handle, _P(cuda_stream)))

  def synchronize(self):
    check(self.lib.wb2_synchronize(self.handle))

  @property
  def launch_count(self) -> int:
    return int(self.lib.wb2_launch_count(self.handle))

  def malloc(self, nbytes: int) -> int:
    p = _P()
    check(self.lib.wb2_malloc(self.handle, nbytes, C.byref(p)))
    return p.value

  def free(self, ptr: int):
    check(self.lib.wb2_free(self.handle, _P(ptr)))

  def host_alloc(self, nbytes: int) -> int:
    p = _P()
    check(self.lib.wb2_host_alloc(self.handle, nbytes, C.byref(p)))
    return p.value

  def host_free(self, ptr: int):
    check(self.lib.wb2_host_free(self.handle, _P(ptr)))

  def pinned_empty(self, shape, dtype) -> np.ndarray:
    """NumPy array backed by pinned host memory (freed with the context)."""
    dtype = np.dtype(dtype)
    n = int(np.prod(shape)) * dtype.itemsize
    ptr = self.host_alloc(max(n, 1))
    buf = (C.c_char * max(n, 1)).from_address(ptr)
    arr = np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape)))
    return arr.reshape(shape)

  def pinned_result(self, shape, dtype) -> np.ndarray:
    """Pinned host array for a result that the library writes with D2H copies.
    A pageable destination costs a page fault per 4 KB on top of the driver's
    bounce copy (measured: 385 MB of spectra took ~100 ms, as long as the
    6 GB of input); pinning a fresh buffer per call costs about the same.
    Buffers therefore come from a per-context pool and RETURN to it when the
    array (and every view of it) is garbage collected, so a chunk loop pays
    the pinning once.  Falls back to pageable memory for small results."""
    dtype = np.dtype(dtype)
    n = int(np.prod(shape)) * dtype.itemsize
    if n < (4 << 20):
      return np.empty(shape, dtype=dtype)
    cap = 1 << max(22, (n - 1).bit_length())  # size classes: powers of two
    pool = self._pinned_pool.setdefault(cap, [])
    ptr = pool.pop() if pool else self.host_alloc(cap)
    buf = (C.c_char * n).from_address(ptr)
    buf._wb2_block = _PinnedBlock(self, ptr, cap)  # lives as long as the array
    return np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(
        shape)

  def _release_pinned(self, ptr: int, cap: int):
    if self._closed:
      return  # the context is gone: a result that outlived it keeps its buffer
    pool = self._pinned_pool.setdefault(cap, [])
    held = sum(len(v) * k for k, v in self._pinned_pool.items())
    if held + cap > self._pinned_pool_limit:
      try:
        self.host_free(ptr)
      except Exception:  # pylint: disable=broad-except
        pass
    else:
      pool.append(ptr)

  def to_device(self, a: np.ndarray) -> int:
    a = np.ascontiguousarray(a)
    p = self.malloc(a.nbytes)
    check(self.lib.wb2_memcpy_h2d(self.handle, _P(p), _P(a.ctypes.data),
                                  a.nbytes))
    return p

  def from_device(self, ptr: int, shape, dtype) -> np.ndarray:
    out = np.empty(shape, dtype=dtype)
    check(self.lib.wb2_memcpy_d2h(self.handle, _P(out.ctypes.data), _P(ptr),
                                  out.nbytes))
    return out

  # -- slab cache / transfer accounting of the *_host entries -------------------
  def set_slab_cache(self, nbytes: int):
    check(self.lib.wb2_set_slab_cache(self.handle, int(nbytes)))
    self._slab_cache_bytes = int(nbytes)

  def slab_cache(self, nbytes: Optional[int] = None):
    """`with ctx.slab_cache(nbytes):` -- keeps the truth / climatology slabs of
    the *_host entries resident in HBM inside the block (LRU, keyed by host
    address; the host arrays must not change meanwhile) and drops them on
    exit.  Default size: 30 % of the free device memory, at most 48 GiB.
    Re-entrant: an enclosing scope's cache is kept."""
    return _SlabCacheScope(self, nbytes)

  def transfer_stats(self) -> dict:
    f = self.lib.wb2_transfer_stats
    return {'h2d_bytes': int(f(self.handle, 0)),
            'd2h_bytes': int(f(self.handle, 1)),
            'cache_hits': int(f(self.handle, 2)),
            'cache_misses': int(f(self.handle, 3))}

  def reset_transfer_stats(self):
    check(self.lib.wb2_reset_transfer_stats(self.handle))

  # -- K1 ---------------------------------------------------------------------
  def det_metrics(self, f: int, t: int, c: Optional[int], dtype: int,
                  off_f: np.ndarray, off_t: np.ndarray,
                  off_c: Optional[np.ndarray], weights: 'WeightSpec',
                  skipna: bool, out: int, host: bool = False):
    """f/t/c/out are raw addresses (device, or host when host=True)."""
    nfield = int(off_f.size)
    w = weights.as_struct()
    fn = self.lib.wb2_det_metrics_host if host else self.lib.wb2_det_metrics
    check(fn(self.handle, _P(f), _P(t), _P(c) if c else None, dtype, nfield,
             _as_ptr(off_f, C.c_int64), _as_ptr(off_t, C.c_int64),
             _as_ptr(off_c, C.c_int64) if off_c is not None else None,
             C.byref(w), int(bool(skipna)), _P(out)))

  def det_metrics_vector(self, fu, fv, tu, tv, dtype, off_fu, off_fv, off_tu,
                         off_tv, weights: 'WeightSpec', skipna: bool, out: int):
    w = weights.as_struct()
    check(self.lib.wb2_det_metrics_vector(
        self.handle, _P(fu), _P(fv), _P(tu), _P(tv), dtype, int(off_fu.size),
        _as_ptr(off_fu, C.c_int64), _as_ptr(off_fv, C.c_int64),
        _as_ptr(off_tu, C.c_int64), _as_ptr(off_tv, C.c_int64), C.byref(w),
        int(bool(skipna)), _P(out)))

  # -- K2 ---------------------------------------------------------------------
  def ens_metrics(self, x: int, t: int, dtype: int, nmember: int,
                  member_stride: int, off_x: np.ndarray, off_t: np.ndarray,
                  weights: 'WeightSpec', skipna: bool, out: int):
    w = weights.as_struct()
    check(self.lib.wb2_ens_metrics(
        self.handle, _P(x), _P(t), dtype, int(nmember), int(member_stride),
        int(off_x.size), _as_ptr(off_x, C.c_int64), _as_ptr(off_t, C.c_int64),
        C.byref(w), int(bool(skipna)), _P(out)))

  def ens_metrics_host(self, x: int, t: int, nmember: int, member_stride: int,
                       off_x: np.ndarray, off_t: np.ndarray,
                       weights: 'WeightSpec', skipna: bool, out: int):
    """x / t / out are HOST addresses (wb2_ens_metrics_host)."""
    w = weights.as_struct()
    check(self.lib.wb2_ens_metrics_host(
        self.handle, _P(x), _P(t), F32, int(nmember), int(member_stride),
        int(off_x.size), _as_ptr(off_x, C.c_int64), _as_ptr(off_t, C.c_int64),
        C.byref(w), int(bool(skipna)), _P(out)))

  # -- K3 ---------------------------------------------------------------------
  def energy_score(self, x: int, t: int, dtype: int, nmember: int,
                   member_stride: int, off_x: np.ndarray, off_t: np.ndarray,
                   weights: 'WeightSpec', out: int):
    w = weights.as_struct()
    check(self.lib.wb2_energy_score(
        self.handle, _P(x), _P(t), dtype, int(nmember), int(member_stride),
        int(off_x.size), _as_ptr(off_x, C.c_int64), _as_ptr(off_t, C.c_int64),
        C.byref(w), _P(out)))

  # -- K6 ---------------------------------------------------------------------
  def det_maps(self, f: int, t: int, dtype: int, stat: int, nout: int,
               ngroup: int, off_f: np.ndarray, off_t: np.ndarray, nrow: int,
               ncol: int, row_stride: int, skipna: bool, out: int):
    assert off_f.size == nout * ngroup and off_t.size == nout * ngroup
    check(self.lib.wb2_det_maps(
        self.handle, _P(f), _P(t), dtype, int(stat), int(nout), int(ngroup),
        _as_ptr(off_f, C.c_int64), _as_ptr(off_t, C.c_int64), int(nrow),
        int(ncol), int(row_stride), int(bool(skipna)), _P(out)))

  def ens_maps(self, x: int, t: int, dtype: int, nmember: int,
               member_stride: int, nout: int, ngroup: int, off_x: np.ndarray,
               off_t: np.ndarray, nrow: int, ncol: int, row_stride: int,
               stat_mask: int, skipna: bool, out: int):
    assert off_x.size == nout * ngroup and off_t.size == nout * ngroup
    check(self.lib.wb2_ens_maps(
        self.handle, _P(x), _P(t), dtype, int(nmember), int(member_stride),
        int(nout), int(ngroup), _as_ptr(off_x, C.c_int64),
        _as_ptr(off_t, C.c_int64), int(nrow), int(ncol), int(row_stride),
        int(stat_mask), int(bool(skipna)), _P(out)))

  # -- K7 ---------------------------------------------------------------------
  @staticmethod
  def _threshold_args(nthreshold, thr_a, off_a, thr_b, off_b, z):
    zz = None if z is None else np.ascontiguousarray(z, dtype=np.float64)
    return (int(nthreshold), _P(thr_a) if thr_a else None,
            _as_ptr(off_a, C.c_int64) if off_a is not None else None,
            _P(thr_b) if thr_b else None,
            _as_ptr(off_b, C.c_int64) if off_b is not None else None,
            _as_ptr(zz, C.c_double) if zz is not None else None), zz

  def ens_threshold_metrics(self, x: int, t: int, nmember: int,
                            member_stride: int, off_x: np.ndarray,
                            off_t: np.ndarray, nthreshold: int, thr_a: int,
                            off_a: np.ndarray, thr_b: Optional[int],
                            off_b: Optional[np.ndarray],
                            z: Optional[np.ndarray], weights: 'WeightSpec',
                            skipna: bool, out: int):
    w = weights.as_struct()
    targs, keep = self._threshold_args(nthreshold, thr_a, off_a, thr_b, off_b,
                                       z)
    check(self.lib.wb2_ens_threshold_metrics(
        self.handle, _P(x), _P(t), F32, int(nmember), int(member_stride),
        int(off_x.size), _as_ptr(off_x, C.c_int64), _as_ptr(off_t, C.c_int64),
        *targs, C.byref(w), int(bool(skipna)), _P(out)))
    del keep

  def ens_threshold_maps(self, x: int, t: int, nmember: int,
                         member_stride: int, nout: int, ngroup: int,
                         off_x: np.ndarray, off_t: np.ndarray, nthreshold: int,
                         thr_a: int, off_a: np.ndarray, thr_b: Optional[int],
                         off_b: Optional[np.ndarray], z: Optional[np.ndarray],
                         nrow: int, ncol: int, row_stride: int, stat: int,
                         skipna: bool, out: int):
    assert off_x.size == nout * ngroup and off_t.size == nout * ngroup
    targs, keep = self._threshold_args(nthreshold, thr_a, off_a, thr_b, off_b,
                                       z)
    check(self.lib.wb2_ens_threshold_maps(
        self.handle, _P(x), _P(t), F32, int(nmember), int(member_stride),
        int(nout), int(ngroup), _as_ptr(off_x, C.c_int64),
        _as_ptr(off_t, C.c_int64), *targs, int(nrow), int(ncol),
        int(row_stride), int(stat), int(bool(skipna)), _P(out)))
    del keep

  def gaussian_metrics(self, mean: int, std: int, t: int, off_mean: np.ndarray,
                       off_std: np.ndarray, off_t: np.ndarray, nthreshold: int,
                       thr_a: Optional[int], off_a: Optional[np.ndarray],
                       thr_b: Optional[int], off_b: Optional[np.ndarray],
                       z: Optional[np.ndarray], weights: 'WeightSpec',
                       skipna: bool, out: int):
    w = weights.as_struct()
    targs, keep = self._threshold_args(nthreshold, thr_a, off_a, thr_b, off_b,
                                       z)
    check(self.lib.wb2_gaussian_metrics(
        self.handle, _P(mean), _P(std), _P(t), F32, int(off_mean.size),
        _as_ptr(off_mean, C.c_int64), _as_ptr(off_std, C.c_int64),
        _as_ptr(off_t, C.c_int64), *targs, C.byref(w), int(bool(skipna)),
        _P(out)))
    del keep

  # -- K5 ---------------------------------------------------------------------
  def regrid_conservative(self, src: int, dst: int, nfield: int,
                          src_stride: int, dst_stride: int, lon_w: 'CsrSpec',
                          lat_w: 'CsrSpec'):
    a, b = lon_w.as_struct(), lat_w.as_struct()
    check(self.lib.wb2_regrid_conservative(
        self.handle, _P(src), _P(dst), int(nfield), int(src_stride),
        int(dst_stride), C.byref(a), C.byref(b)))

  def regrid_conservative_host(self, src: int, dst: int, nfield: int,
                               src_stride: int, dst_stride: int,
                               lon_w: 'CsrSpec', lat_w: 'CsrSpec'):
    """src / dst are HOST addresses (wb2_regrid_conservative_host)."""
    a, b = lon_w.as_struct(), lat_w.as_struct()
    check(self.lib.wb2_regrid_conservative_host(
        self.handle, _P(src), _P(dst), int(nfield), int(src_stride),
        int(dst_stride), C.byref(a), C.byref(b)))

  # -- derived variables -------------------------------------------------------
  def wind_speed(self, u: int, v: int, out: int, n: int):
    check(self.lib.wb2_wind_speed(self.handle, _P(u), _P(v), _P(out), int(n)))

  def wind_dynamics(self, kind: int, u: Optional[int], v: Optional[int],
                    z: Optional[int], nouter: int, nlev: int, nlat: int,
                    nlon: int, lat_stride: int, lon_stride: int,
                    lat_coef: np.ndarray, lat_uniform: bool,
                    lon_coef: np.ndarray, lon_uniform: bool,
                    cos_lat: np.ndarray, coriolis: Optional[np.ndarray],
                    pressure: Optional[np.ndarray], out: int):
    """u / v / z / out are DEVICE addresses (wb2_wind_dynamics); the tables
    are host float64 arrays (see the header for their layout)."""
    tabs = [None if a is None else np.ascontiguousarray(a, dtype=np.float64)
            for a in (lat_coef, lon_coef, cos_lat, coriolis, pressure)]
    lc, oc, cs, cor, pres = tabs
    check(self.lib.wb2_wind_dynamics(
        self.handle, int(kind), _P(u) if u else None, _P(v) if v else None,
        _P(z) if z else None, int(nouter), int(nlev), int(nlat), int(nlon),
        int(lat_stride), int(lon_stride), _as_ptr(lc, C.c_double),
        int(bool(lat_uniform)), _as_ptr(oc, C.c_double),
        int(bool(lon_uniform)), _as_ptr(cs, C.c_double),
        _as_ptr(cor, C.c_double), _as_ptr(pres, C.c_double),
        _P(out) if out else None))
    del tabs

  def column_integral(self, kind: int, dtype: int, q: Optional[int],
                      u: Optional[int], v: Optional[int], nouter: int,
                      outer_stride: int, nlev: int, ninner: int, nlon: int,
                      lon_stride: int, weight: Optional[np.ndarray], out: int):
    """q / u / v / out are DEVICE addresses (wb2_column_integral); weight
    is the host float64 table w_k = 0.5 * (level[k+1] - level[k])."""
    w = (None if weight is None
         else np.ascontiguousarray(weight, dtype=np.float64))
    check(self.lib.wb2_column_integral(
        self.handle, int(kind), int(dtype), *(_P(p) if p else None
                                              for p in (q, u, v)),
        int(nouter), int(outer_stride), int(nlev), int(ninner), int(nlon),
        int(lon_stride), _as_ptr(w, C.c_double), _P(out) if out else None))
    del w

  def lapse_rate(self, dtype: int, t: int, z: int, nouter: int, nlev: int,
                 ninner: int, coef: np.ndarray, uniform: bool, out: int):
    """t / z / out are DEVICE addresses (wb2_lapse_rate); coef is the host
    [nlev][3] float64 table of _derived_wind.gradient_table."""
    c = np.ascontiguousarray(coef, dtype=np.float64)
    check(self.lib.wb2_lapse_rate(
        self.handle, int(dtype), _P(t) if t else None, _P(z) if z else None,
        int(nouter), int(nlev), int(ninner), _as_ptr(c, C.c_double),
        int(bool(uniform)), _P(out) if out else None))
    del c

  def relative_humidity(self, dtype: int, out_dtype: int, t: int, q: int,
                        nouter: int, npres: int, ninner: int,
                        pressure: np.ndarray, out: int):
    """t / q / out are DEVICE addresses (wb2_relative_humidity); pressure is
    the host [npres] float64 table of the pressure coordinate."""
    p = np.ascontiguousarray(pressure, dtype=np.float64)
    check(self.lib.wb2_relative_humidity(
        self.handle, int(dtype), int(out_dtype), _P(t) if t else None,
        _P(q) if q else None, int(nouter), int(npres), int(ninner),
        _as_ptr(p, C.c_double), _P(out) if out else None))
    del p

  def ens_mean(self, x: int, nmember: int, member_stride: int,
               off_x: np.ndarray, slab: int, skipna: bool, out: int):
    off_x = np.ascontiguousarray(off_x, dtype=np.int64)
    check(self.lib.wb2_ens_mean(
        self.handle, _P(x), int(nmember), int(member_stride), int(off_x.size),
        _as_ptr(off_x, C.c_int64), int(slab), int(bool(skipna)), _P(out)))

  def spectrum_interp(self, spec: int, nfield: int, nrow: int, nk: int,
                      freq_table: np.ndarray, freqs: np.ndarray, out: int):
    """freq_table: [nrow][nk] increasing frequencies of every latitude row."""
    step = np.ascontiguousarray(freq_table, dtype=np.float64)
    assert step.shape == (nrow, nk)
    fr = np.ascontiguousarray(freqs, dtype=np.float64)
    check(self.lib.wb2_spectrum_interp(
        self.handle, _P(spec), int(nfield), int(nrow), int(nk),
        _as_ptr(step, C.c_double), int(fr.size), _as_ptr(fr, C.c_double),
        _P(out)))

  # -- day-of-year climatology -----------------------------------------------
  @staticmethod
  def _climatology_args(plan: 'ClimatologyPlan'):
    return (int(plan.nres), _as_ptr(plan.res_start, C.c_int64),
            _as_ptr(plan.res_count, C.c_int32), int(plan.nhour),
            int(plan.nday), int(plan.nitem), _as_ptr(plan.items, C.c_int64),
            _as_ptr(plan.fill, C.c_int64), _as_ptr(plan.hour_nday, C.c_int32),
            _as_ptr(plan.out_row, C.c_int32), int(plan.nday_out),
            int(plan.window_size), int(plan.method))

  def climatology(self, x: int, dtype: int, ntime: int, ncell: int,
                  plan: 'ClimatologyPlan', mean: Optional[int],
                  std: Optional[int]):
    """x / mean / std are DEVICE addresses (wb2_climatology)."""
    check(self.lib.wb2_climatology(
        self.handle, _P(x), dtype, int(ntime), int(ncell),
        *self._climatology_args(plan), _P(mean) if mean else None,
        _P(std) if std else None))

  def climatology_host(self, x: int, dtype: int, ntime: int, ncell: int,
                       plan: 'ClimatologyPlan', budget: int,
                       mean: Optional[int], std: Optional[int]):
    """x / mean / std are HOST addresses (wb2_climatology_host)."""
    check(self.lib.wb2_climatology_host(
        self.handle, _P(x), dtype, int(ntime), int(ncell),
        *self._climatology_args(plan), int(budget),
        _P(mean) if mean else None, _P(std) if std else None))

  @staticmethod
  def _quantile_args(quantiles, seeps_threshold: Optional[float]):
    q = np.ascontiguousarray(quantiles, dtype=np.float64)
    return (int(q.size), _as_ptr(q, C.c_double),
            int(seeps_threshold is not None),
            float(seeps_threshold if seeps_threshold is not None else 0.0)), q

  def climatology_quantile(self, x: int, dtype: int, ntime: int, ncell: int,
                           plan: 'ClimatologyPlan', quantiles,
                           seeps_threshold: Optional[float], out: int,
                           dry_fraction: Optional[int]):
    """x / out / dry_fraction are DEVICE addresses (wb2_climatology_quantile);
    seeps_threshold None computes the quantiles, else the SEEPS pair."""
    args, keep = self._quantile_args(quantiles, seeps_threshold)
    check(self.lib.wb2_climatology_quantile(
        self.handle, _P(x), dtype, int(ntime), int(ncell),
        *self._climatology_args(plan)[:-1], *args, _P(out),
        _P(dry_fraction) if dry_fraction else None))
    del keep

  def climatology_quantile_host(self, x: int, dtype: int, ntime: int,
                                ncell: int, plan: 'ClimatologyPlan', quantiles,
                                seeps_threshold: Optional[float], budget: int,
                                out: int, dry_fraction: Optional[int]):
    """x / out / dry_fraction are HOST addresses
    (wb2_climatology_quantile_host)."""
    args, keep = self._quantile_args(quantiles, seeps_threshold)
    check(self.lib.wb2_climatology_quantile_host(
        self.handle, _P(x), dtype, int(ntime), int(ncell),
        *self._climatology_args(plan)[:-1], *args, int(budget), _P(out),
        _P(dry_fraction) if dry_fraction else None))
    del keep

  # -- time resampling / rolling windows ---------------------------------------
  @staticmethod
  def _time_window_args(bin_start, bin_count):
    s = None if bin_start is None else np.ascontiguousarray(bin_start,
                                                            dtype=np.int64)
    c = None if bin_count is None else np.ascontiguousarray(bin_count,
                                                            dtype=np.int32)
    nbin = s.size if s is not None else (c.size if c is not None else 0)
    return (int(nbin), _as_ptr(s, C.c_int64), _as_ptr(c, C.c_int32)), (s, c)

  def time_window_stats(self, x: int, dtype: int, nouter: int, ntime: int,
                        ninner: int, bin_start, bin_count, window: int,
                        skipna: bool, mean: Optional[int], min: Optional[int],  # pylint: disable=redefined-builtin
                        max: Optional[int], sum: Optional[int]):  # pylint: disable=redefined-builtin
    """x and the outputs are DEVICE addresses (wb2_time_window_stats);
    bin_start / bin_count host arrays (resample) or None (rolling window)."""
    args, keep = self._time_window_args(bin_start, bin_count)
    check(self.lib.wb2_time_window_stats(
        self.handle, _P(x), dtype, int(nouter), int(ntime), int(ninner), *args,
        int(window), int(bool(skipna)), *(_P(p) if p else None
                                          for p in (mean, min, max, sum))))
    del keep

  def time_window_stats_host(self, x: int, dtype: int, nouter: int,
                             ntime: int, ninner: int, bin_start, bin_count,
                             window: int, skipna: bool, budget: int,
                             mean: Optional[int], min: Optional[int],  # pylint: disable=redefined-builtin
                             max: Optional[int], sum: Optional[int]):  # pylint: disable=redefined-builtin
    """x and the outputs are HOST addresses (wb2_time_window_stats_host)."""
    args, keep = self._time_window_args(bin_start, bin_count)
    check(self.lib.wb2_time_window_stats_host(
        self.handle, _P(x), dtype, int(nouter), int(ntime), int(ninner), *args,
        int(window), int(bool(skipna)), int(budget),
        *(_P(p) if p else None for p in (mean, min, max, sum))))
    del keep

  # -- precipitation accumulations over lead time -----------------------------
  def precip_accumulation(self, x: int, dtype: int, nouter: int, ntime: int,
                          ninner: int, window: int, clamp_negative: bool,
                          out: int):
    """x and out are DEVICE addresses (wb2_precip_accumulation)."""
    check(self.lib.wb2_precip_accumulation(
        self.handle, _P(x) if x else None, dtype, int(nouter), int(ntime),
        int(ninner), int(window), int(bool(clamp_negative)),
        _P(out) if out else None))

  def precip_accumulation_host(self, x: int, dtype: int, nouter: int,
                               ntime: int, ninner: int, window: int,
                               clamp_negative: bool, budget: int, out: int):
    """x and out are HOST addresses (wb2_precip_accumulation_host)."""
    check(self.lib.wb2_precip_accumulation_host(
        self.handle, _P(x) if x else None, dtype, int(nouter), int(ntime),
        int(ninner), int(window), int(bool(clamp_negative)), int(budget),
        _P(out) if out else None))

  # -- quantiles over a sample axis --------------------------------------------
  @staticmethod
  def _quantile_list(quantiles):
    if quantiles is None:
      return 0, None, None
    q = np.ascontiguousarray(quantiles, dtype=np.float64).reshape(-1)
    return int(q.size), _as_ptr(q, C.c_double), q

  def quantile(self, x: int, dtype: int, nouter: int, nsample: int,
               ninner: int, quantiles, skipna: bool, out: int,
               nquantile: Optional[int] = None):
    """x and out are DEVICE addresses (wb2_quantile); quantiles a host
    sequence of float64 (`nquantile` overrides its length)."""
    nq, qp, keep = self._quantile_list(quantiles)
    check(self.lib.wb2_quantile(
        self.handle, _P(x) if x else None, dtype, int(nouter), int(nsample),
        int(ninner), nq if nquantile is None else int(nquantile), qp,
        int(bool(skipna)), _P(out) if out else None))
    del keep

  def quantile_host(self, x: int, dtype: int, nouter: int, nsample: int,
                    ninner: int, quantiles, skipna: bool, budget: int,
                    out: int, nquantile: Optional[int] = None):
    """x and out are HOST addresses (wb2_quantile_host)."""
    nq, qp, keep = self._quantile_list(quantiles)
    check(self.lib.wb2_quantile_host(
        self.handle, _P(x) if x else None, dtype, int(nouter), int(nsample),
        int(ninner), nq if nquantile is None else int(nquantile), qp,
        int(bool(skipna)), int(budget), _P(out) if out else None))
    del keep

  # -- means and raw moments over reduced dims ---------------------------------
  @staticmethod
  def _average_args(shape, weights):
    if len(shape) != 5:
      raise ValueError(f'shape must be (k0, r0, k1, r1, k2) (got {shape})')
    if weights is None:
      return [int(s) for s in shape], None, None
    w = np.ascontiguousarray(weights, dtype=np.float64).reshape(-1)
    return [int(s) for s in shape], _as_ptr(w, C.c_double), w

  def average(self, x: int, dtype: int, shape, skipna: bool, mean: int = 0,
              mean_sq: int = 0, frac: int = 0, weights=None, wdiv: int = 1,
              wlen: Optional[int] = None):
    """x and the outputs are DEVICE addresses (wb2_average); `shape` is the
    canonical (k0, r0, k1, r1, k2); `weights` a host float64 table indexed by
    (s / wdiv) % wlen (`wlen` defaults to its length); 0 skips an output."""
    sh, wp, keep = self._average_args(shape, weights)
    wl = (0 if keep is None else keep.size) if wlen is None else int(wlen)
    check(self.lib.wb2_average(
        self.handle, _P(x) if x else None, dtype, *sh, wp, int(wdiv), wl,
        int(bool(skipna)), _P(mean) if mean else None,
        _P(mean_sq) if mean_sq else None, _P(frac) if frac else None))
    del keep

  def average_host(self, x: int, dtype: int, shape, skipna: bool, budget: int,
                   mean: int = 0, mean_sq: int = 0, frac: int = 0,
                   weights=None, wdiv: int = 1, wlen: Optional[int] = None):
    """x and the outputs are HOST addresses (wb2_average_host)."""
    sh, wp, keep = self._average_args(shape, weights)
    wl = (0 if keep is None else keep.size) if wlen is None else int(wlen)
    check(self.lib.wb2_average_host(
        self.handle, _P(x) if x else None, dtype, *sh, wp, int(wdiv), wl,
        int(bool(skipna)), int(budget), _P(mean) if mean else None,
        _P(mean_sq) if mean_sq else None, _P(frac) if frac else None))
    del keep

  # -- slab gather (reindexing in time) ---------------------------------------
  def slab_gather(self, src: int, src_dtype: int, src_elems: int, slab: int,
                  nslab: int, offsets, out: int, out_dtype: int = F32):
    """src and out are DEVICE addresses (wb2_slab_gather); offsets a host
    int64 table of nslab source offsets, negative for a NaN slab."""
    off = np.ascontiguousarray(offsets, dtype=np.int64).reshape(-1)
    check(self.lib.wb2_slab_gather(
        self.handle, _P(src) if src else None, int(src_dtype), int(src_elems),
        int(slab), int(nslab), _as_ptr(off, C.c_int64), _P(out) if out else None,
        int(out_dtype)))

  def slab_gather_host(self, src: int, src_dtype: int, src_elems: int,
                       slab: int, nslab: int, offsets, budget: int, out: int,
                       out_dtype: int = F32):
    """src and out are HOST addresses (wb2_slab_gather_host)."""
    off = np.ascontiguousarray(offsets, dtype=np.int64).reshape(-1)
    check(self.lib.wb2_slab_gather_host(
        self.handle, _P(src) if src else None, int(src_dtype), int(src_elems),
        int(slab), int(nslab), _as_ptr(off, C.c_int64), int(budget),
        _P(out) if out else None, int(out_dtype)))

  # -- K10 --------------------------------------------------------------------
  def rank_histogram(self, x: int, t: int, nmember: int, member_stride: int,
                     nout: int, ngroup: int, off_x: np.ndarray,
                     off_t: np.ndarray, nrow: int, ncol: int, row_stride: int,
                     nbins: int, random_ties: bool, seed: int, out: int):
    assert off_x.size == nout * ngroup and off_t.size == nout * ngroup
    check(self.lib.wb2_rank_histogram(
        self.handle, _P(x), _P(t), int(nmember), int(member_stride),
        int(nout), int(ngroup), _as_ptr(off_x, C.c_int64),
        _as_ptr(off_t, C.c_int64), int(nrow), int(ncol), int(row_stride),
        int(nbins), int(bool(random_ties)), int(seed) & (2**64 - 1), _P(out)))

  # -- K9 ---------------------------------------------------------------------
  def seeps_maps(self, f: int, t: int, wet: int, p1: int, nout: int,
                 ngroup: int, off_f: np.ndarray, off_t: np.ndarray,
                 off_wet_f: np.ndarray, off_wet_t: np.ndarray, nrow: int,
                 ncol: int, row_stride: int, wet_row_stride: int,
                 dry_threshold: float, min_p1: float, max_p1: float,
                 skipna: bool, out: int, *, f_dtype: int = F32,
                 t_dtype: int = F32, wet_dtype: int = F32,
                 p1_dtype: int = F32):
    """K9.  The *_dtype keywords are F32 (the default) or F64, one per
    operand; the three thresholds are Python floats, rounded by the kernel to
    the dtype they are compared in."""
    n = nout * ngroup
    assert off_f.size == n and off_t.size == n
    assert off_wet_f.size == n and off_wet_t.size == n
    check(self.lib.wb2_seeps_maps(
        self.handle, _P(f), int(f_dtype), _P(t), int(t_dtype), _P(wet),
        int(wet_dtype), _P(p1), int(p1_dtype), int(nout), int(ngroup),
        _as_ptr(off_f, C.c_int64), _as_ptr(off_t, C.c_int64),
        _as_ptr(off_wet_f, C.c_int64), _as_ptr(off_wet_t, C.c_int64),
        int(nrow), int(ncol), int(row_stride), int(wet_row_stride),
        float(dry_threshold), float(min_p1), float(max_p1),
        int(bool(skipna)), _P(out)))

  # -- K8 ---------------------------------------------------------------------
  def regrid_gather(self, src: int, dst: int, nfield: int, src_stride: int,
                    dst_stride: int, nsource: int, indices: np.ndarray):
    idx = np.ascontiguousarray(indices, dtype=np.int32)
    check(self.lib.wb2_regrid_gather(
        self.handle, _P(src), _P(dst), int(nfield), int(src_stride),
        int(dst_stride), int(nsource), int(idx.size),
        _as_ptr(idx, C.c_int32)))

  def regrid_bilinear(self, src: int, dst: int, nfield: int, src_stride: int,
                      dst_stride: int, source_shape, lon_taps, lat_taps):
    """lon_taps / lat_taps: (i0, i1, t) arrays per target coordinate."""
    li0, li1, lt = (np.ascontiguousarray(lon_taps[0], np.int32),
                    np.ascontiguousarray(lon_taps[1], np.int32),
                    np.ascontiguousarray(lon_taps[2], np.float32))
    ai0, ai1, at = (np.ascontiguousarray(lat_taps[0], np.int32),
                    np.ascontiguousarray(lat_taps[1], np.int32),
                    np.ascontiguousarray(lat_taps[2], np.float32))
    check(self.lib.wb2_regrid_bilinear(
        self.handle, _P(src), _P(dst), int(nfield), int(src_stride),
        int(dst_stride), int(source_shape[0]), int(source_shape[1]),
        int(li0.size), int(ai0.size), _as_ptr(li0, C.c_int32),
        _as_ptr(li1, C.c_int32), _as_ptr(lt, C.c_float),
        _as_ptr(ai0, C.c_int32), _as_ptr(ai1, C.c_int32),
        _as_ptr(at, C.c_float)))

  # -- K4 ---------------------------------------------------------------------
  def zonal_spectrum(self, x: int, nfield: int, nrow: int, ncol: int,
                     scale: np.ndarray, out: int, accumulate: bool = False,
                     nfield_out: int = 0):
    scale = np.ascontiguousarray(scale, dtype=np.float64)
    check(self.lib.wb2_zonal_spectrum(
        self.handle, _P(x), int(nfield), int(nrow), int(ncol),
        _as_ptr(scale, C.c_double), _P(out), int(bool(accumulate)),
        int(nfield_out)))


  def zonal_spectrum_host(self, x: int, nfield: int, nrow: int, ncol: int,
                          scale: np.ndarray, out: int, accumulate: bool = False,
                          nfield_out: int = 0):
    """x / out are HOST addresses (wb2_zonal_spectrum_host)."""
    scale = np.ascontiguousarray(scale, dtype=np.float64)
    check(self.lib.wb2_zonal_spectrum_host(
        self.handle, _P(x), int(nfield), int(nrow), int(ncol),
        _as_ptr(scale, C.c_double), _P(out), int(bool(accumulate)),
        int(nfield_out)))

  def zonal_spectrum_latsum_host(self, x: int, nfield: int, nrow: int,
                                 ncol: int, scale: np.ndarray, out: int,
                                 nfield_out: int):
    scale = np.ascontiguousarray(scale, dtype=np.float64)
    check(self.lib.wb2_zonal_spectrum_latsum_host(
        self.handle, _P(x), int(nfield), int(nrow), int(ncol),
        _as_ptr(scale, C.c_double), _P(out), int(nfield_out)))

  def zonal_spectrum_latsum(self, x: int, nfield: int, nrow: int, ncol: int,
                            scale: np.ndarray, out: int, nfield_out: int):
    """out[slot][k] = sum over the slot's fields and over rows of
    scale[row] * spectrum (scale = circumference * latitude weight)."""
    scale = np.ascontiguousarray(scale, dtype=np.float64)
    check(self.lib.wb2_zonal_spectrum_latsum(
        self.handle, _P(x), int(nfield), int(nrow), int(ncol),
        _as_ptr(scale, C.c_double), _P(out), int(nfield_out)))


class _PinnedBlock:
  """Returns a pinned buffer to its context's pool when the last array backed
  by it goes away."""

  def __init__(self, ctx: 'Context', ptr: int, cap: int):
    self.ctx, self.ptr, self.cap = ctx, ptr, cap

  def __del__(self):
    try:
      self.ctx._release_pinned(self.ptr, self.cap)  # pylint: disable=protected-access
    except Exception:  # pylint: disable=broad-except
      pass


class _SlabCacheScope:
  """Context manager behind Context.slab_cache()."""

  def __init__(self, ctx: 'Context', nbytes: Optional[int]):
    self.ctx, self.nbytes, self.owner = ctx, nbytes, False

  def __enter__(self):
    ctx = self.ctx
    if getattr(ctx, '_slab_cache_bytes', 0) > 0:
      return ctx  # an enclosing scope already holds a cache
    nbytes = self.nbytes
    if nbytes is None:
      nbytes = default_slab_cache_bytes(ctx.device)
    if nbytes > 0:
      ctx.set_slab_cache(nbytes)
      self.owner = True
    return ctx

  def __exit__(self, *exc):
    if self.owner:
      self.ctx.set_slab_cache(0)
    return False


def default_slab_cache_bytes(device: int) -> int:
  """30 % of the free device memory, capped at 48 GiB (WB2_SLAB_CACHE_MB
  overrides; 0 disables)."""
  env = os.environ.get('WB2_SLAB_CACHE_MB')
  if env is not None:
    return int(env) << 20
  try:
    import torch  # pylint: disable=import-outside-toplevel
    free, _ = torch.cuda.mem_get_info(device)
  except Exception:  # pylint: disable=broad-except
    free = 16 << 30
  return int(min(0.3 * free, 48 << 30))


class WeightSpec:
  """Host-side owner of the arrays a wb2_weights struct points to."""

  def __init__(self, nrow, ncol, row_w, seg_start, seg_w, col_w=None,
               cell_w_dev: Optional[int] = None, zero_skip=False,
               row_stride=None):
    self.nrow, self.ncol = int(nrow), int(ncol)
    self.row_stride = int(row_stride if row_stride is not None else ncol)
    self.row_w = np.ascontiguousarray(row_w, dtype=np.float64).reshape(
        -1, self.nrow)
    self.nregion = self.row_w.shape[0]
    self.seg_start = np.ascontiguousarray(seg_start, dtype=np.int32)
    self.nseg = self.seg_start.size - 1
    self.seg_w = np.ascontiguousarray(seg_w, dtype=np.float64).reshape(
        self.nregion, self.nseg)
    self.col_w = (None if col_w is None else
                  np.ascontiguousarray(col_w, dtype=np.float32))
    self.cell_w_dev = cell_w_dev
    self.zero_skip = bool(zero_skip)

  def as_struct(self) -> Weights:
    w = Weights()
    w.nrow, w.ncol, w.row_stride = self.nrow, self.ncol, self.row_stride
    w.nregion, w.nseg = self.nregion, self.nseg
    w.row_w = _as_ptr(self.row_w, C.c_double)
    w.seg_start = _as_ptr(self.seg_start, C.c_int32)
    w.seg_w = _as_ptr(self.seg_w, C.c_double)
    w.col_w = _as_ptr(self.col_w, C.c_float) if self.col_w is not None else None
    w.cell_w = self.cell_w_dev
    w.zero_skip = int(self.zero_skip)
    return w


class ClimatologyPlan:
  """Host-side owner of the index tables of wb2_climatology (see the header):
  which time steps (or resampled days) feed every (hour, day slot)."""

  def __init__(self, items, fill, hour_nday, out_row, nday_out, window_size,
               method, res_start=None, res_count=None):
    self.items = np.ascontiguousarray(items, dtype=np.int64)
    self.nhour, self.nday, self.nitem = self.items.shape
    self.fill = (np.ascontiguousarray(fill, dtype=np.int64)
                 if fill is not None else np.full((self.nhour, self.nitem), -1,
                                                  np.int64))
    self.hour_nday = np.ascontiguousarray(hour_nday, dtype=np.int32)
    self.out_row = np.ascontiguousarray(out_row, dtype=np.int32)
    self.nday_out = int(nday_out)
    self.window_size = int(window_size)
    self.method = int(method)  # 0 explicit, 1 fast
    if res_start is None:
      self.res_start = np.zeros(1, np.int64)
      self.res_count = np.zeros(1, np.int32)
      self.nres = 0
    else:
      self.res_start = np.ascontiguousarray(res_start, dtype=np.int64)
      self.res_count = np.ascontiguousarray(res_count, dtype=np.int32)
      self.nres = int(self.res_start.size)


class CsrSpec:
  """Host-side owner of a wb2_csr (banded regridding weights)."""

  def __init__(self, dense: np.ndarray):
    dense = np.asarray(dense, dtype=np.float32)
    self.n_tgt, self.n_src = dense.shape
    nan_row = np.isnan(dense).any(axis=1)
    row_ptr = [0]
    cols, vals = [], []
    for i in range(self.n_tgt):
      if not nan_row[i]:
        nz = np.nonzero(dense[i])[0]
        cols.append(nz)
        vals.append(dense[i, nz])
      row_ptr.append(row_ptr[-1] + (0 if nan_row[i] else nz.size))
    self.row_ptr = np.asarray(row_ptr, dtype=np.int32)
    self.col_idx = (np.concatenate(cols).astype(np.int32) if cols
                    else np.zeros(0, np.int32))
    self.val = (np.concatenate(vals).astype(np.float32) if vals
                else np.zeros(0, np.float32))
    if self.col_idx.size == 0:  # keep pointers valid
      self.col_idx = np.zeros(1, np.int32)
      self.val = np.zeros(1, np.float32)
    self.nan_row = nan_row.astype(np.uint8)

  def as_struct(self) -> Csr:
    s = Csr()
    s.n_src, s.n_tgt = self.n_src, self.n_tgt
    s.row_ptr = _as_ptr(self.row_ptr, C.c_int32)
    s.col_idx = _as_ptr(self.col_idx, C.c_int32)
    s.val = _as_ptr(self.val, C.c_float)
    s.nan_row = _as_ptr(self.nan_row, C.c_uint8)
    return s


_default_ctx = {}
_ctx_lock = threading.Lock()


def default_context(device: Optional[int] = None) -> Context:
  """Process-wide context per device (device defaults to LOCAL_RANK or 0)."""
  if device is None:
    device = int(os.environ.get('WB2_DEVICE', os.environ.get('LOCAL_RANK', 0)))
  with _ctx_lock:
    ctx = _default_ctx.get(device)
    if ctx is None:
      ctx = Context(device)
      _default_ctx[device] = ctx
    return ctx

// Quantiles over a sample axis: wb2_quantile (device series) and
// wb2_quantile_host (NumPy / memmap series streamed in bands).
//
// Replaces xarray's Dataset.quantile(q, dim, skipna) with method='linear', the
// whole computation of scripts/compute_quantiles.py:168-183.  x is
// [nouter][nsample][ninner] and is read in place; out is float64
// [nquantile][nouter][ninner].  Numerics are numpy's np.quantile /
// np.nanquantile bit for bit (include/wb2b200.h and DESIGN.md section 8f pin
// the six steps): order statistics s[i], s[j] of the m valid samples,
// d = T(s[j] - s[i]) and one separately rounded float64 lerp.
//
// Two paths, chosen from nsample alone:
//   short (nsample <= 64)  quantile_short_kernel: a CTA stages 128 cells x n
//                          samples in shared memory with coalesced loads, one
//                          thread per cell sorts its samples in registers with
//                          the Batcher network of the next generated size (NaN
//                          and padding are +Inf) and writes them back to its
//                          own column, from which the quantiles read s[i], s[j].
//   long                   quantile_long_kernel: one warp per cell selects the
//                          ranks it needs by an MSD radix select on
//                          order-preserving integer keys, 8 bits per pass, with a
//                          per-warp shared histogram.  All ranks share the first
//                          histogram; s[i + 1] comes from one counting pass after
//                          s[i].  When a tile of 128 B of cells x n samples fits
//                          in shared memory it is staged once (kStaged); else
//                          each pass reads the cell from global memory, 8
//                          neighbouring cells per CTA so the CTA's warps share
//                          sectors through L1.
#include <math_constants.h>

#include <algorithm>
#include <cmath>

#include "stage.cuh"

namespace wb2 {

constexpr int kQsMaxQuantiles = 128;
constexpr int kQsShortMax = 64;                     // largest sort network
constexpr int kQsShortCells = 128;                  // cells (threads) per short CTA
constexpr int kQsShortPitch = kQsShortCells + 1;    // conflict-free both ways
constexpr int kQsWarps = 8;
constexpr int kQsThreads = kQsWarps * 32;
constexpr int kQsBins = 256;
constexpr size_t kQsHistBytes = size_t(kQsWarps) * 2 * kQsBins * sizeof(unsigned long long);
constexpr size_t kQsSmemLimit = 227 * 1024;         // H100 opt-in shared memory per block

struct QsList {
  double q[kQsMaxQuantiles];
};

// Order-preserving keys: the float bits with the sign bit flipped (positive)
// or every bit flipped (negative), so -Inf < ... < -0 < +0 < ... < +Inf as
// unsigned integers.  Every NaN maps to the largest key, above +Inf.
template <typename T>
struct QsKey;
template <>
struct QsKey<float> {
  using U = uint32_t;
  static constexpr int kBits = 32;
  static __device__ __forceinline__ U key(float v) {
    const U b = __float_as_uint(v);
    return v != v ? ~U(0) : b ^ ((b >> 31) ? ~U(0) : U(1) << 31);
  }
  static __device__ __forceinline__ float value(U k) {
    return __uint_as_float((k >> 31) ? k ^ (U(1) << 31) : ~k);
  }
  static __device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
};
template <>
struct QsKey<double> {
  using U = unsigned long long;
  static constexpr int kBits = 64;
  static __device__ __forceinline__ U key(double v) {
    const U b = static_cast<U>(__double_as_longlong(v));
    return v != v ? ~U(0) : b ^ ((b >> 63) ? ~U(0) : U(1) << 63);
  }
  static __device__ __forceinline__ double value(U k) {
    return __longlong_as_double(static_cast<long long>((k >> 63) ? k ^ (U(1) << 63) : ~k));
  }
  static __device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
};

// Steps 3-5 of the contract: the indices and weight of quantile q among m
// sorted valid samples (numpy's _get_indexes / _get_gamma for 'linear') ...
__device__ __forceinline__ void qs_index(int64_t m, double q, int64_t* i, int64_t* j,
                                         double* g) {
  const double v = __dmul_rn(double(m - 1), q);
  if (v >= double(m - 1)) {
    *i = *j = m - 1;
    *g = __dadd_rn(v, 1.0);
  } else {
    const double f = floor(v);
    *i = int64_t(f);
    *j = *i + 1;
    *g = __dsub_rn(v, f);
  }
}
// ... and numpy's _lerp: the difference rounded in T, then float64.
template <typename T>
__device__ __forceinline__ double qs_lerp(T a, T b, double g) {
  const double d = double(QsKey<T>::sub(b, a));
  return g < 0.5 ? __dadd_rn(double(a), __dmul_rn(d, g))
                 : __dsub_rn(double(b), __dmul_rn(d, __dsub_rn(1.0, g)));
}

// Copies the samples of the w cells c0 .. c0+w-1 (flat [nouter][ninner] order)
// of x [nouter][n][ninner] into tile[s * pitch + (cell - c0)].  Wide inner
// axes: the cells of one outer index are a run of columns, read row by row.
// Narrow ones (ninner < 32): the tile's outer slabs are one contiguous span,
// read linearly and filtered.  Consecutive threads read consecutive addresses
// either way.  Block-wide; the caller synchronises.
template <typename T, int kThreads>
__device__ __forceinline__ void qs_stage(const T* __restrict__ x, int n, int64_t ninner, int64_t c0, int w,
                         int pitch, T* tile) {
  if (ninner >= 32) {
    for (int c = 0; c < w;) {
      const int64_t cell = c0 + c;
      const int64_t o = cell / ninner, i0 = cell - o * ninner;
      const int run = int(std::min<int64_t>(w - c, ninner - i0));
      const T* src = x + o * n * ninner + i0;
      for (int e = threadIdx.x; e < n * run; e += kThreads) {
        const int s = e / run, r = e - s * run;
        tile[s * pitch + c + r] = ldg_stream(src + int64_t(s) * ninner + r);
      }
      c += run;
    }
  } else {
    const int ni = int(ninner);
    const int64_t o0 = c0 / ninner;
    const int lo = int(c0 - o0 * ninner);            // first cell's column in slab o0
    const int slab = n * ni;
    const int span = int((c0 + w - 1) / ninner - o0 + 1) * slab;
    const T* src = x + o0 * slab;
    for (int e = threadIdx.x; e < span; e += kThreads) {
      const int ob = e / slab, r = e - ob * slab;
      const int s = r / ni, i = r - s * ni;
      const int c = ob * ni + i - lo;
      if (c >= 0 && c < w) tile[s * pitch + c] = ldg_stream(src + e);
    }
  }
}

// ---- short axes: register sorting networks ---------------------------------
template <typename T>
__device__ __forceinline__ void qs_ce(T& a, T& b) {
  // exact exchange (no min / max): the sorted column is a permutation of the
  // samples, +-0 included
  const bool sw = b < a;
  const T lo = sw ? b : a;
  b = sw ? a : b;
  a = lo;
}
#define CE(a, b) qs_ce(v[a], v[b]);
#define CE2(a, b) qs_ce(v[a], v[b]); qs_ce(v[(a) + 1], v[(b) + 1]);
#include "sort_networks.inc"
#undef CE
#undef CE2

template <typename T, int N>
__global__ void __launch_bounds__(kQsShortCells)
    quantile_short_kernel(const T* __restrict__ x, int n, int64_t ninner, int64_t ncell,
                          int nq, const QsList ql, int skipna, double* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char qs_smem[];
  T* tile = reinterpret_cast<T*>(qs_smem);  // [n][kQsShortPitch]
  const int64_t c0 = int64_t(blockIdx.x) * kQsShortCells;
  const int w = int(std::min<int64_t>(ncell - c0, kQsShortCells));
  qs_stage<T, kQsShortCells>(x, n, ninner, c0, w, kQsShortPitch, tile);
  __syncthreads();
  const int c = threadIdx.x;
  if (c >= w) return;
  const T inf = T(CUDART_INF);
  T v[N];
  int nnan = 0;
#pragma unroll
  for (int k = 0; k < N; ++k) {
    T e = k < n ? tile[k * kQsShortPitch + c] : inf;
    if (e != e) {
      ++nnan;
      e = inf;
    }
    v[k] = e;
  }
  SortNet<N>::run(v);
  // the first m = n - nnan entries are the valid samples in order: padding,
  // NaN and real +Inf are equal keys at the end
#pragma unroll
  for (int k = 0; k < N; ++k)
    if (k < n) tile[k * kQsShortPitch + c] = v[k];
  const int m = n - nnan;
  const bool none = m == 0 || (!skipna && nnan > 0);
  double* oc = out + c0 + c;
  for (int k = 0; k < nq; ++k) {
    double r = CUDART_NAN;
    if (!none) {
      int64_t i, j;
      double g;
      qs_index(m, ql.q[k], &i, &j, &g);
      r = qs_lerp(tile[int(i) * kQsShortPitch + c], tile[int(j) * kQsShortPitch + c], g);
    }
    oc[int64_t(k) * ncell] = r;
  }
}

// ---- long axes: radix select -----------------------------------------------
// The samples of one cell: a staged tile column or a strided global series.
template <typename T, bool kStaged>
struct QsSrc {
  const T* p;
  int64_t stride;
  __device__ __forceinline__ T operator[](int64_t s) const {
    return kStaged ? p[s * stride] : __ldg(p + s * stride);
  }
};

// Histogram h[256] of digit (key >> shift) & 255 over the cell's keys whose
// bits above shift + 8 equal `prefix` (every key when `all`), counting equal
// digits of a warp step once with match.any.  Returns this lane's NaN count.
template <typename T, bool kStaged>
__device__ __forceinline__ int64_t qs_hist(const QsSrc<T, kStaged>& src, int64_t n, int shift,
                           typename QsKey<T>::U prefix, bool all, unsigned long long* h,
                           int lane) {
  using U = typename QsKey<T>::U;
  for (int b = lane; b < kQsBins; b += 32) h[b] = 0;
  __syncwarp();
  int64_t nnan = 0;
  for (int64_t s0 = 0; s0 < n; s0 += 32) {
    const int64_t s = s0 + lane;
    int d = -1;
    if (s < n) {
      const U k = QsKey<T>::key(src[s]);
      nnan += k == ~U(0);
      if (all || (k >> (shift + 8)) == prefix) d = int(k >> shift) & (kQsBins - 1);
    }
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    if (d >= 0 && lane == __ffs(peers) - 1)
      atomicAdd(h + d, static_cast<unsigned long long>(__popc(peers)));
  }
  __syncwarp();
  return nnan;
}

// The bin of h that holds rank *r (0-based); *r becomes the rank inside it.
__device__ __forceinline__ int qs_bucket(const unsigned long long* h, int64_t* r, int lane) {
  unsigned long long c[kQsBins / 32], sum = 0;
#pragma unroll
  for (int t = 0; t < kQsBins / 32; ++t) {
    c[t] = h[lane * (kQsBins / 32) + t];
    sum += c[t];
  }
  unsigned long long inc = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long u = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += u;
  }
  const unsigned long long rr = static_cast<unsigned long long>(*r), exc = inc - sum;
  const int src = __ffs(__ballot_sync(0xffffffffu, rr >= exc && rr < inc)) - 1;
  int b = 0;
  unsigned long long below = exc;
  if (lane == src) {
#pragma unroll
    for (int t = 0; t < kQsBins / 32; ++t) {
      if (rr < below + c[t]) {
        b = lane * (kQsBins / 32) + t;
        break;
      }
      below += c[t];
    }
  }
  b = __shfl_sync(0xffffffffu, b, src);
  below = __shfl_sync(0xffffffffu, below, src);
  *r = static_cast<int64_t>(rr - below);
  return b;
}

template <typename T, bool kStaged>
__global__ void __launch_bounds__(kQsThreads, 1)
    quantile_long_kernel(const T* __restrict__ x, int64_t n, int64_t ninner, int64_t ncell,
                         int cells, int pitch, int nq, const QsList ql, int skipna,
                         double* __restrict__ out) {
  using K = QsKey<T>;
  using U = typename K::U;
  extern __shared__ __align__(16) unsigned char qs_smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long* h1 = reinterpret_cast<unsigned long long*>(qs_smem) + warp * 2 * kQsBins;
  unsigned long long* h2 = h1 + kQsBins;
  T* tile = reinterpret_cast<T*>(qs_smem + kQsHistBytes);  // [n][pitch] when staged
  const int64_t c0 = int64_t(blockIdx.x) * cells;
  const int w = int(std::min<int64_t>(ncell - c0, cells));
  if (kStaged) {
    qs_stage<T, kQsThreads>(x, int(n), ninner, c0, w, pitch, tile);
    __syncthreads();
  }
  for (int c = warp; c < w; c += kQsWarps) {
    const int64_t cell = c0 + c;
    QsSrc<T, kStaged> src;
    if (kStaged) {
      src.p = tile + c;
      src.stride = pitch;
    } else {
      const int64_t o = cell / ninner;
      src.p = x + o * n * ninner + (cell - o * ninner);
      src.stride = ninner;
    }
    int64_t nnan = qs_hist<T, kStaged>(src, n, K::kBits - 8, 0, true, h1, lane);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nnan += __shfl_xor_sync(0xffffffffu, nnan, o);
    const int64_t m = n - nnan;
    const bool none = m == 0 || (!skipna && nnan > 0);
    int64_t last = -1;
    U ki = 0, kj = 0;
    for (int k = 0; k < nq; ++k) {
      double r = CUDART_NAN;
      if (!none) {
        int64_t i, j;
        double g;
        qs_index(m, ql.q[k], &i, &j, &g);
        if (i != last) {  // j follows from i: i + 1, or i itself at the top
          int64_t rank = i;
          U prefix = U(qs_bucket(h1, &rank, lane));
          for (int shift = K::kBits - 16; shift >= 0; shift -= 8) {
            qs_hist<T, kStaged>(src, n, shift, prefix, false, h2, lane);
            prefix = (prefix << 8) | U(qs_bucket(h2, &rank, lane));
          }
          ki = prefix;
          kj = ki;
          if (j != i) {  // s[i + 1]: s[i] again if more than i + 1 keys are <= it
            int64_t le = 0;
            U mn = ~U(0);
            for (int64_t s = lane; s < n; s += 32) {
              const U kk = K::key(src[s]);
              le += kk <= ki;
              if (kk > ki && kk < mn) mn = kk;
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
              le += __shfl_xor_sync(0xffffffffu, le, o);
              const U u = __shfl_xor_sync(0xffffffffu, mn, o);
              mn = u < mn ? u : mn;
            }
            kj = le > j ? ki : mn;
          }
          last = i;
        }
        r = qs_lerp(K::value(ki), K::value(kj), g);
      }
      if (lane == 0) out[int64_t(k) * ncell + cell] = r;
    }
  }
}

// ---- launch ------------------------------------------------------------------
template <typename T>
constexpr int qs_long_cells() { return 128 / int(sizeof(T)); }  // 128 B of cells

// The largest nsample whose long-path tile is staged in shared memory.
template <typename T>
constexpr int64_t qs_max_staged() {
  return int64_t((kQsSmemLimit - kQsHistBytes) / ((qs_long_cells<T>() + 1) * sizeof(T)));
}

static int qs_validate(int dtype, int64_t nouter, int64_t nsample, int64_t ninner,
                       int32_t nquantile, const double* quantiles) {
  WB2_REQUIRE(dtype == WB2_F32 || dtype == WB2_F64,
              "dtype must be WB2_F32 or WB2_F64 (got %d)", dtype);
  WB2_REQUIRE(nsample >= 1, "nsample must be >= 1 (got %lld)",
              static_cast<long long>(nsample));
  WB2_REQUIRE(nouter >= 0 && ninner >= 0, "nouter and ninner must be >= 0");
  WB2_REQUIRE(nquantile >= 1 && nquantile <= kQsMaxQuantiles,
              "nquantile must be in 1..%d (got %d)", kQsMaxQuantiles, nquantile);
  WB2_REQUIRE(quantiles != nullptr, "quantiles is NULL");
  for (int k = 0; k < nquantile; ++k)
    WB2_REQUIRE(quantiles[k] >= 0.0 && quantiles[k] <= 1.0,
                "quantiles[%d] = %g is not in [0, 1]", k, quantiles[k]);
  WB2_REQUIRE(nouter == 0 || ninner == 0 || nouter * ninner / kQsWarps < 0x7fffffff,
              "too many cells (nouter * ninner) for the quantile kernels' grid");
  return WB2_OK;
}

template <typename T, int N>
static int qs_launch_short(wb2_ctx* ctx, const T* x, int n, int64_t ninner, int64_t ncell,
                           int nq, const QsList& ql, int skipna, double* out) {
  const size_t smem = size_t(n) * kQsShortPitch * sizeof(T);
  return launch_kernel(ctx, quantile_short_kernel<T, N>,
                       dim3(static_cast<unsigned>((ncell + kQsShortCells - 1) / kQsShortCells)),
                       kQsShortCells, smem, x, n, ninner, ncell, nq, ql, skipna, out);
}

template <typename T>
static int qs_launch(wb2_ctx* ctx, const T* x, int64_t nouter, int64_t n, int64_t ninner,
                     int nq, const QsList& ql, int skipna, double* out) {
  const int64_t ncell = nouter * ninner;
  if (n <= kQsShortMax) {
    const int ni = int(n);
    int rc;
    if (n <= 2) rc = qs_launch_short<T, 2>(ctx, x, ni, ninner, ncell, nq, ql, skipna, out);
    else if (n <= 3) rc = qs_launch_short<T, 3>(ctx, x, ni, ninner, ncell, nq, ql, skipna, out);
    else if (n <= 4) rc = qs_launch_short<T, 4>(ctx, x, ni, ninner, ncell, nq, ql, skipna, out);
    else if (n <= 5) rc = qs_launch_short<T, 5>(ctx, x, ni, ninner, ncell, nq, ql, skipna, out);
    else if (n <= 8) rc = qs_launch_short<T, 8>(ctx, x, ni, ninner, ncell, nq, ql, skipna, out);
    else if (n <= 10) rc = qs_launch_short<T, 10>(ctx, x, ni, ninner, ncell, nq, ql, skipna, out);
    else if (n <= 16) rc = qs_launch_short<T, 16>(ctx, x, ni, ninner, ncell, nq, ql, skipna, out);
    else if (n <= 20) rc = qs_launch_short<T, 20>(ctx, x, ni, ninner, ncell, nq, ql, skipna, out);
    else if (n <= 32) rc = qs_launch_short<T, 32>(ctx, x, ni, ninner, ncell, nq, ql, skipna, out);
    else if (n <= 50) rc = qs_launch_short<T, 50>(ctx, x, ni, ninner, ncell, nq, ql, skipna, out);
    else rc = qs_launch_short<T, 64>(ctx, x, ni, ninner, ncell, nq, ql, skipna, out);
    WB2_TRY(rc);
  } else if (n <= qs_max_staged<T>()) {
    constexpr int cells = qs_long_cells<T>();
    const size_t smem = kQsHistBytes + size_t(n) * (cells + 1) * sizeof(T);
    WB2_TRY(launch_kernel(ctx, quantile_long_kernel<T, true>,
                          dim3(static_cast<unsigned>((ncell + cells - 1) / cells)), kQsThreads,
                          smem, x, n, ninner, ncell, cells, cells + 1, nq, ql, skipna, out));
  } else {
    WB2_TRY(launch_kernel(ctx, quantile_long_kernel<T, false>,
                          dim3(static_cast<unsigned>((ncell + kQsWarps - 1) / kQsWarps)),
                          kQsThreads, kQsHistBytes, x, n, ninner, ncell, kQsWarps, 0, nq, ql,
                          skipna, out));
  }
  ctx->launches += 1;
  return WB2_OK;
}

static int qs_launch_any(wb2_ctx* ctx, int dtype, const void* x, int64_t nouter, int64_t n,
                         int64_t ninner, int nq, const QsList& ql, int skipna, double* out) {
  if (dtype == WB2_F32)
    return qs_launch(ctx, static_cast<const float*>(x), nouter, n, ninner, nq, ql, skipna, out);
  return qs_launch(ctx, static_cast<const double*>(x), nouter, n, ninner, nq, ql, skipna, out);
}

static QsList qs_list(int32_t nquantile, const double* quantiles) {
  QsList ql{};
  std::copy(quantiles, quantiles + nquantile, ql.q);
  return ql;
}

}  // namespace wb2

using namespace wb2;

extern "C" {

int wb2_quantile(wb2_ctx* ctx, const void* x, int dtype, int64_t nouter, int64_t nsample,
                 int64_t ninner, int32_t nquantile, const double* quantiles, int skipna,
                 double* out) {
  WB2_NVTX("wb2_quantile");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_TRY(qs_validate(dtype, nouter, nsample, ninner, nquantile, quantiles));
  if (nouter == 0 || ninner == 0) return WB2_OK;
  WB2_REQUIRE(x != nullptr, "x is NULL");
  WB2_REQUIRE(out != nullptr, "out is NULL");
  DeviceGuard guard(ctx->device);
  return qs_launch_any(ctx, dtype, x, nouter, nsample, ninner, nquantile,
                       qs_list(nquantile, quantiles), skipna ? 1 : 0, out);
}

int wb2_quantile_host(wb2_ctx* ctx, const void* x, int dtype, int64_t nouter, int64_t nsample,
                      int64_t ninner, int32_t nquantile, const double* quantiles, int skipna,
                      size_t budget, double* out) {
  WB2_NVTX("wb2_quantile_host");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_TRY(qs_validate(dtype, nouter, nsample, ninner, nquantile, quantiles));
  if (nouter == 0 || ninner == 0) return WB2_OK;
  WB2_REQUIRE(x != nullptr, "x is NULL");
  WB2_REQUIRE(out != nullptr, "out is NULL");
  DeviceGuard guard(ctx->device);
  const QsList ql = qs_list(nquantile, quantiles);
  char* const out_host[1] = {reinterpret_cast<char*>(out)};
  return stream_series_bands(
      ctx, x, dtype == WB2_F32 ? 4 : 8, sizeof(double), nouter, nsample, ninner, nquantile,
      true, out_host, 1, budget, [&](const void* in, int64_t k, int64_t n, void* const* dev_out) {
        return qs_launch_any(ctx, dtype, in, k, nsample, n, nquantile, ql, skipna ? 1 : 0,
                             static_cast<double*>(dev_out[0]));
      });
}

}  // extern "C"

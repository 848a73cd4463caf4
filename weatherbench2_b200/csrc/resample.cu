// Time resampling and rolling windows: wb2_time_window_stats (device series)
// and wb2_time_window_stats_host (NumPy / memmap series streamed in bands).
//
// Replaces xarray's resample(...).mean/min/max/sum and rolling(...,
// min_periods=None).mean/min/max/sum, the computation of
// scripts/resample_in_time.py.  The series is [nouter][ntime][ninner] and is
// read in place; every requested statistic comes out of one read.
//
// Semantics (the header and DESIGN.md section 8c pin them):
//   case                     mean / min / max / sum
//   resample, skipna 0       any NaN in the bin -> NaN
//   resample, skipna 1       NaN skipped; all-NaN non-empty bin: mean / min /
//                            max NaN, sum 0 (nansum)
//   resample, empty bin      NaN for every statistic, sum included
//   rolling (window w)       output t reduces [t-w+1, t]; NaN when t < w-1 or
//                            when any value of the window is NaN, whatever
//                            skipna is; w > ntime: all NaN
//   +-Inf                    NumPy float64 over the window: mean([1, inf]) =
//                            inf, inf + -inf = nan, finite again once the Inf
//                            has left the window
// Mean and sum accumulate in float64; min and max are compared in the input's
// precision, so each is bit-equal to one of the window's values.
//
// Disjoint bins (resample), and rolling windows wider than kRollMaxWindow:
//   time_bins_kernel, one thread per (outer, inner) cell walks a chunk of the
//   bins; a warp's loads are coalesced over inner cells and each thread has
//   kLoadBatch loads of a bin in flight before it accumulates them.
// Rolling, w <= kRollMaxWindow:
//   time_rolling_kernel, a CTA owns 128 B of inner cells (32 float / 16
//   double) x kRollBlock consecutive outputs and stages those rows plus the
//   w-1 halo rows once in shared memory, so HBM reads are (B + w - 1) / B of
//   the input.  The CTA's threads split the outputs into segments per cell.
//   Sums slide over float64 sums of the finite values with separate counts of
//   NaN, +Inf and -Inf (a running sum that subtracted an Inf would stay NaN).
//   Min / max use van Herk / Gil-Werman: suffix extrema of blocks of w rows
//   (shared memory) and running prefix extrema, O(1) per output.
#include <math_constants.h>

#include <algorithm>

#include "stage.cuh"

namespace wb2 {

constexpr int kTwThreads = 256;
constexpr int kLoadBatch = 8;        // loads in flight per thread
constexpr int kRollBlock = 256;      // outputs per CTA of the staged rolling kernel
constexpr int kRollMaxWindow = 168;  // one week of hourly data

template <typename T>
struct TwOut {
  T* mean;
  T* min;
  T* max;
  T* sum;
};

template <typename T>
__device__ __forceinline__ T tw_inf() {
  return T(CUDART_INF);
}

template <typename T>
__global__ void __launch_bounds__(kTwThreads)
    time_bins_kernel(const T* __restrict__ x, int64_t ncellall, int64_t ntime, int64_t ninner,
                     int64_t nout, const int64_t* __restrict__ bstart,
                     const int32_t* __restrict__ bcount, int32_t window, int skipna,
                     int64_t per_chunk, TwOut<T> out) {
  const int64_t gid = int64_t(blockIdx.x) * kTwThreads + threadIdx.x;
  if (gid >= ncellall) return;
  const int64_t o = gid / ninner, i = gid - o * ninner;
  const T* xc = x + o * ntime * ninner + i;
  const int64_t b0 = int64_t(blockIdx.y) * per_chunk;
  const int64_t b1 = b0 + per_chunk < nout ? b0 + per_chunk : nout;
  const T qnan = T(CUDART_NAN);
  for (int64_t b = b0; b < b1; ++b) {
    int64_t s;
    int32_t c;
    if (bstart != nullptr) {
      s = bstart[b];
      c = bcount[b];
    } else {  // rolling window ending at b
      s = b - window + 1;
      c = s >= 0 ? window : 0;
    }
    double acc = 0.0;
    int32_t nval = 0;
    bool nan = false;
    T lo = tw_inf<T>(), hi = -tw_inf<T>();
    for (int32_t j0 = 0; j0 < c; j0 += kLoadBatch) {
      T v[kLoadBatch];
#pragma unroll
      for (int k = 0; k < kLoadBatch; ++k)
        v[k] = j0 + k < c ? ldg_stream(xc + (s + j0 + k) * ninner) : qnan;
#pragma unroll
      for (int k = 0; k < kLoadBatch; ++k) {
        if (j0 + k < c) {
          if (v[k] != v[k]) {
            nan = true;
          } else {
            acc += double(v[k]);
            ++nval;
            lo = v[k] < lo ? v[k] : lo;
            hi = v[k] > hi ? v[k] : hi;
          }
        }
      }
    }
    const bool nan_all = c == 0 || (nan && !skipna);
    const bool none = nan_all || nval == 0;
    const int64_t oi = (o * nout + b) * ninner + i;
    if (out.mean) out.mean[oi] = none ? qnan : T(acc / double(nval));
    if (out.min) out.min[oi] = none ? qnan : lo;
    if (out.max) out.max[oi] = none ? qnan : hi;
    if (out.sum) out.sum[oi] = nan_all ? qnan : T(acc);
  }
}

template <typename T>
struct RollShape {
  static constexpr int kCells = 128 / int(sizeof(T));  // one 128-B row per CTA
  static constexpr int kSegs = kTwThreads / kCells;    // output segments per cell
  static constexpr int kSeg = kRollBlock / kSegs;      // outputs per segment
};

template <typename T>
__global__ void __launch_bounds__(kTwThreads)
    time_rolling_kernel(const T* __restrict__ x, int64_t ntime, int64_t ninner,
                        int64_t ntile, int32_t w, TwOut<T> out) {
  using S = RollShape<T>;
  extern __shared__ __align__(16) unsigned char tw_smem[];
  const int rows = kRollBlock + w - 1;
  T* xs = reinterpret_cast<T*>(tw_smem);  // [rows][kCells], row j = step t0 - w + 1 + j
  T* hlo = xs + rows * S::kCells;          // [kRollBlock][kCells] block suffix extrema
  T* hhi = hlo + kRollBlock * S::kCells;
  const int64_t o = blockIdx.x / ntile;
  const int64_t cell = (blockIdx.x - o * ntile) * S::kCells + threadIdx.x % S::kCells;
  const int cl = threadIdx.x % S::kCells, sg = threadIdx.x / S::kCells;
  const bool live = cell < ninner;
  const T* xc = x + o * ntime * ninner + (live ? cell : 0);
  const int64_t t0 = int64_t(blockIdx.y) * kRollBlock;
  const int64_t g0 = t0 - w + 1;
  const T qnan = T(CUDART_NAN);

  // stage the block and its halo; steps outside [0, ntime) read as NaN, which
  // makes the first w-1 outputs NaN
  for (int j0 = sg; j0 < rows; j0 += S::kSegs * kLoadBatch) {
    T v[kLoadBatch];
#pragma unroll
    for (int k = 0; k < kLoadBatch; ++k) {
      const int j = j0 + k * S::kSegs;
      const int64_t g = g0 + j;
      v[k] = live && j < rows && g >= 0 && g < ntime ? ldg_stream(xc + g * ninner) : qnan;
    }
#pragma unroll
    for (int k = 0; k < kLoadBatch; ++k) {
      const int j = j0 + k * S::kSegs;
      if (j < rows) xs[j * S::kCells + cl] = v[k];
    }
  }
  __syncthreads();

  // this thread's segment: outputs a .. a+n-1 (tile rows), output t's window is
  // staged rows [t, t + w)
  const int a = sg * S::kSeg;
  const int64_t left = ntime - t0 - a;
  const int n = left < S::kSeg ? int(left) : S::kSeg;
  if (!live || n <= 0) return;
  const bool ext = out.min || out.max;
  if (ext) {  // suffix extrema of blocks of w rows aligned at a (rows beyond the
              // segment only feed the blocks that start inside it)
    for (int b = a; b < a + n; b += w) {
      T lo = tw_inf<T>(), hi = -tw_inf<T>();
      for (int j = b + w - 1; j >= b; --j) {
        const T v = xs[j * S::kCells + cl];
        lo = v < lo ? v : lo;
        hi = v > hi ? v : hi;
        if (j < a + n) {
          hlo[j * S::kCells + cl] = lo;
          hhi[j * S::kCells + cl] = hi;
        }
      }
    }
  }
  double acc = 0.0;
  int nnan = 0, npos = 0, nneg = 0;
  auto add = [&](T v, int sign) {
    if (v != v) nnan += sign;
    else if (v == tw_inf<T>()) npos += sign;
    else if (v == -tw_inf<T>()) nneg += sign;
    else acc += sign > 0 ? double(v) : -double(v);
  };
  for (int j = a; j < a + w - 1; ++j) add(xs[j * S::kCells + cl], 1);
  T glo = tw_inf<T>(), ghi = -tw_inf<T>();  // prefix extrema of the block of row t+w-1
  int phase = w - 1;                         // (t + w - 1 - a) mod w
  for (int t = a; t < a + n; ++t) {
    const T v = xs[(t + w - 1) * S::kCells + cl];
    add(v, 1);
    if (ext) {
      if (phase == 0) {
        glo = v;
        ghi = v;
      } else {
        glo = v < glo ? v : glo;
        ghi = v > ghi ? v : ghi;
      }
      phase = phase + 1 == w ? 0 : phase + 1;
    }
    const int64_t oi = (o * ntime + t0 + t) * ninner + cell;
    const bool nan = nnan > 0;
    const double s = nan || (npos && nneg) ? double(CUDART_NAN)
                     : npos               ? double(CUDART_INF)
                     : nneg               ? -double(CUDART_INF)
                                          : acc;
    if (out.mean) out.mean[oi] = T(s / double(w));
    if (out.sum) out.sum[oi] = T(s);
    if (ext) {
      const T hl = hlo[t * S::kCells + cl], hh = hhi[t * S::kCells + cl];
      if (out.min) out.min[oi] = nan ? qnan : (hl < glo ? hl : glo);
      if (out.max) out.max[oi] = nan ? qnan : (hh > ghi ? hh : ghi);
    }
    add(xs[t * S::kCells + cl], -1);
  }
}

// Staged rolling path: bytes of dynamic shared memory.
template <typename T>
static size_t tw_roll_smem(int32_t w, bool ext) {
  constexpr int c = RollShape<T>::kCells;
  return (size_t(kRollBlock) + w - 1) * c * sizeof(T) +
         (ext ? 2 * size_t(kRollBlock) * c * sizeof(T) : 0);
}

static int tw_validate(int dtype, int64_t nouter, int64_t ntime, int64_t ninner, int64_t nbin,
                       const int64_t* bin_start, const int32_t* bin_count, int32_t window,
                       const void* mean, const void* min, const void* max, const void* sum) {
  WB2_REQUIRE(dtype == WB2_F32 || dtype == WB2_F64,
              "dtype must be WB2_F32 or WB2_F64 (got %d)", dtype);
  WB2_REQUIRE(nouter >= 0 && ntime >= 0 && ninner >= 0,
              "nouter / ntime / ninner must be >= 0");
  WB2_REQUIRE(window >= 0, "window must be >= 0 (got %d)", window);
  const bool bins = bin_start != nullptr || bin_count != nullptr;
  WB2_REQUIRE(bins != (window > 0),
              "exactly one of the bins (bin_start / bin_count) or window must be given");
  WB2_REQUIRE(mean || min || max || sum, "none of mean / min / max / sum requested");
  if (!bins) {
    WB2_REQUIRE(nbin == 0, "nbin must be 0 with a window (got %lld)",
                static_cast<long long>(nbin));
    WB2_REQUIRE(window > kRollMaxWindow || (ntime + kRollBlock - 1) / kRollBlock <= 65535,
                "ntime = %lld is too long for the rolling kernel's grid",
                static_cast<long long>(ntime));
    return WB2_OK;
  }
  WB2_REQUIRE(bin_start && bin_count, "bin_start and bin_count must both be given");
  WB2_REQUIRE(nbin >= 0, "nbin must be >= 0 (got %lld)", static_cast<long long>(nbin));
  int64_t end = 0;  // first step after the previous bin
  for (int64_t b = 0; b < nbin; ++b) {
    const long long lb = static_cast<long long>(b);
    WB2_REQUIRE(bin_count[b] >= 0, "bin_count[%lld] = %d < 0", lb, bin_count[b]);
    WB2_REQUIRE(bin_start[b] >= 0 && bin_start[b] <= ntime &&
                    (bin_count[b] == 0 || bin_start[b] < ntime),
                "bin_start[%lld] = %lld out of [0, ntime = %lld)", lb,
                static_cast<long long>(bin_start[b]), static_cast<long long>(ntime));
    WB2_REQUIRE(bin_start[b] + bin_count[b] <= ntime,
                "bin %lld (bin_start %lld, bin_count %d) ends past ntime = %lld", lb,
                static_cast<long long>(bin_start[b]), bin_count[b],
                static_cast<long long>(ntime));
    WB2_REQUIRE(bin_start[b] >= end,
                "bin_start[%lld] = %lld overlaps the previous bin (bins must be "
                "non-decreasing and disjoint)",
                lb, static_cast<long long>(bin_start[b]));
    end = bin_start[b] + bin_count[b];
  }
  return WB2_OK;
}

template <typename T>
static int tw_launch(wb2_ctx* ctx, const T* x, int64_t nouter, int64_t ntime, int64_t ninner,
                     int64_t nbin, const int64_t* d_start, const int32_t* d_count,
                     int32_t window, int skipna, TwOut<T> out) {
  const int64_t nout = window > 0 ? ntime : nbin;
  const int64_t ncell = nouter * ninner;
  if (ncell == 0 || nout == 0) return WB2_OK;
  if (window > 0 && window <= kRollMaxWindow) {
    constexpr int c = RollShape<T>::kCells;
    const int64_t ntile = (ninner + c - 1) / c;
    WB2_REQUIRE(nouter * ntile <= 0x7fffffff, "too many cells for the rolling kernel's grid");
    const size_t smem = tw_roll_smem<T>(window, out.min || out.max);
    WB2_CUDA_TRY(cudaFuncSetAttribute(time_rolling_kernel<T>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
    const dim3 grid(static_cast<unsigned>(nouter * ntile),
                    static_cast<unsigned>((ntime + kRollBlock - 1) / kRollBlock));
    time_rolling_kernel<T><<<grid, kTwThreads, smem, ctx->stream>>>(x, ntime, ninner, ntile,
                                                                    window, out);
  } else {
    const int64_t nblk = (ncell + kTwThreads - 1) / kTwThreads;
    WB2_REQUIRE(nblk <= 0x7fffffff, "too many cells for the resample kernel's grid");
    // split the bins over blockIdx.y until about two waves of threads are resident
    const int64_t want = int64_t(ctx->num_sms) * 2048 * 2;
    int64_t nchunk = std::min<int64_t>((want + ncell - 1) / ncell, std::min<int64_t>(nout, 65535));
    nchunk = std::max<int64_t>(nchunk, 1);
    const int64_t per_chunk = (nout + nchunk - 1) / nchunk;
    nchunk = (nout + per_chunk - 1) / per_chunk;
    const dim3 grid(static_cast<unsigned>(nblk), static_cast<unsigned>(nchunk));
    time_bins_kernel<T><<<grid, kTwThreads, 0, ctx->stream>>>(
        x, ncell, ntime, ninner, nout, d_start, d_count, window, window > 0 ? 0 : skipna,
        per_chunk, out);
  }
  WB2_CUDA_TRY(cudaGetLastError());
  ctx->launches += 1;
  return WB2_OK;
}

static int tw_launch_any(wb2_ctx* ctx, int dtype, const void* x, int64_t nouter, int64_t ntime,
                         int64_t ninner, int64_t nbin, const int64_t* d_start,
                         const int32_t* d_count, int32_t window, int skipna,
                         void* const* out) {
  if (dtype == WB2_F32) {
    const TwOut<float> o{static_cast<float*>(out[0]), static_cast<float*>(out[1]),
                         static_cast<float*>(out[2]), static_cast<float*>(out[3])};
    return tw_launch(ctx, static_cast<const float*>(x), nouter, ntime, ninner, nbin, d_start,
                     d_count, window, skipna, o);
  }
  const TwOut<double> o{static_cast<double*>(out[0]), static_cast<double*>(out[1]),
                        static_cast<double*>(out[2]), static_cast<double*>(out[3])};
  return tw_launch(ctx, static_cast<const double*>(x), nouter, ntime, ninner, nbin, d_start,
                   d_count, window, skipna, o);
}

// Device copy of the bin tables ([start][count] in `blk`), or NULL pointers
// when there are none.
static int tw_upload(wb2_ctx* ctx, int64_t nbin, const int64_t* start, const int32_t* count,
                     DeviceBlock* blk, const int64_t** d_start, const int32_t** d_count) {
  *d_start = nullptr;
  *d_count = nullptr;
  if (nbin == 0 || start == nullptr) return WB2_OK;
  size_t o[2];
  WB2_TRY(upload_parts(ctx, {{start, size_t(nbin) * 8}, {count, size_t(nbin) * 4}}, blk, o));
  *d_start = blk->at<const int64_t>(o[0]);
  *d_count = blk->at<const int32_t>(o[1]);
  return WB2_OK;
}

}  // namespace wb2

using namespace wb2;

extern "C" {

int wb2_time_window_stats(wb2_ctx* ctx, const void* x, int dtype, int64_t nouter, int64_t ntime,
                          int64_t ninner, int64_t nbin, const int64_t* bin_start,
                          const int32_t* bin_count, int32_t window, int skipna, void* mean,
                          void* min, void* max, void* sum) {
  WB2_NVTX("wb2_time_window_stats");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_TRY(tw_validate(dtype, nouter, ntime, ninner, nbin, bin_start, bin_count, window, mean,
                      min, max, sum));
  const int64_t nout = window > 0 ? ntime : nbin;
  if (nouter == 0 || ninner == 0 || nout == 0) return WB2_OK;
  WB2_REQUIRE(x != nullptr, "x is NULL");
  DeviceGuard guard(ctx->device);
  void* const out[4] = {mean, min, max, sum};
  DeviceBlock tables;
  const int64_t* d_start;
  const int32_t* d_count;
  WB2_TRY(tw_upload(ctx, nbin, bin_start, bin_count, &tables, &d_start, &d_count));
  return tw_launch_any(ctx, dtype, x, nouter, ntime, ninner, nbin, d_start, d_count, window,
                       skipna, out);
}

int wb2_time_window_stats_host(wb2_ctx* ctx, const void* x, int dtype, int64_t nouter,
                               int64_t ntime, int64_t ninner, int64_t nbin,
                               const int64_t* bin_start, const int32_t* bin_count,
                               int32_t window, int skipna, size_t budget, void* mean, void* min,
                               void* max, void* sum) {
  WB2_NVTX("wb2_time_window_stats_host");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_TRY(tw_validate(dtype, nouter, ntime, ninner, nbin, bin_start, bin_count, window, mean,
                      min, max, sum));
  const int64_t nout = window > 0 ? ntime : nbin;
  if (nouter == 0 || ninner == 0 || nout == 0) return WB2_OK;
  WB2_REQUIRE(x != nullptr, "x is NULL");
  DeviceGuard guard(ctx->device);
  char* const out_host[4] = {static_cast<char*>(mean), static_cast<char*>(min),
                             static_cast<char*>(max), static_cast<char*>(sum)};
  DeviceBlock tables;
  const int64_t* d_start;
  const int32_t* d_count;
  WB2_TRY(tw_upload(ctx, nbin, bin_start, bin_count, &tables, &d_start, &d_count));
  const size_t es = dtype == WB2_F32 ? 4 : 8;
  return stream_series_bands(
      ctx, x, es, es, nouter, ntime, ninner, nout, false, out_host, 4, budget,
      [&](const void* in, int64_t k, int64_t n, void* const* out) {
        return tw_launch_any(ctx, dtype, in, k, ntime, n, nbin, d_start, d_count, window,
                             skipna, out);
      });
}

}  // extern "C"

// Precipitation accumulations over lead time: wb2_precip_accumulation (device
// series) and wb2_precip_accumulation_host (NumPy / memmap series streamed in
// bands).
//
// Replaces PrecipitationAccumulation.compute (weatherbench2/
// derived_variables.py:471-528): tp.diff(lead), rolling(lead: w).sum(), the
// relu and a NaN step in front.  The series is [nouter][ntime][ninner] and is
// read in place.  Numerics (the header and DESIGN.md section 8e pin them):
//   out[t] = NaN                                  t < w
//   d[k]   = T(x[k] - x[k-1])                     rounded in the data type T
//   s      = d[t-w+1] + d[t-w+2] + ... + d[t]     float64, oldest first
//   out[t] = T(s), and +0 where T(s) < 0 with clamp_negative (NaN and -0 kept)
// NaN and +-Inf follow from that arithmetic; correctly rounded intrinsics
// keep the compiler from contracting or reassociating any of it.
//
// precip_kernel: a CTA owns 128 B of inner cells (32 float / 16 double) x
// kPaBlock consecutive outputs.  It stages the kPaBlock + w rows
// x[t0-w .. t0+kPaBlock-1] once in shared memory (steps outside the series
// read as NaN, which makes the first w outputs NaN), turns them into
// differences in place, and each thread sums the windows of its outputs from
// shared memory.  HBM traffic: the input once plus w halo rows per block, and
// the output once; no difference array is written.
#include <math_constants.h>

#include <algorithm>

#include "stage.cuh"

namespace wb2 {

constexpr int kPaThreads = 256;
constexpr int kPaBlock = 256;        // outputs per CTA
constexpr int kPaMaxWindow = 1024;   // staged rows: (256 + 1024) x 128 B = 160 KB
constexpr int kPaLoadBatch = 8;      // staging loads in flight per thread
constexpr int kPaIlp = 4;            // windows summed side by side per thread

template <typename T>
struct PaShape {
  static constexpr int kCells = 128 / int(sizeof(T));  // one 128-B row per CTA
  static constexpr int kSegs = kPaThreads / kCells;    // output segments per cell
  static constexpr int kSeg = kPaBlock / kSegs;        // outputs per segment
  static_assert(kSeg % kPaIlp == 0, "segments split into groups of kPaIlp");
};

__device__ __forceinline__ float pa_sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double pa_sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float pa_round(double s, float) { return __double2float_rn(s); }
__device__ __forceinline__ double pa_round(double s, double) { return s; }

template <typename T>
__global__ void __launch_bounds__(kPaThreads)
    precip_kernel(const T* __restrict__ x, int64_t ntime, int64_t ninner, int64_t ntile,
                  int32_t w, int clamp, T* __restrict__ out) {
  using S = PaShape<T>;
  extern __shared__ __align__(16) unsigned char pa_smem[];
  T* xs = reinterpret_cast<T*>(pa_smem);  // [rows][kCells], row j = step t0 - w + j
  const int rows = kPaBlock + w;
  const int64_t o = blockIdx.x / ntile;
  const int64_t cell = (blockIdx.x - o * ntile) * S::kCells + threadIdx.x % S::kCells;
  const int cl = threadIdx.x % S::kCells, sg = threadIdx.x / S::kCells;
  const bool live = cell < ninner;
  const T* xc = x + o * ntime * ninner + (live ? cell : 0);
  const int64_t t0 = int64_t(blockIdx.y) * kPaBlock;
  const int64_t g0 = t0 - w;
  const T qnan = T(CUDART_NAN);

  for (int j0 = sg; j0 < rows; j0 += S::kSegs * kPaLoadBatch) {
    T v[kPaLoadBatch];
#pragma unroll
    for (int k = 0; k < kPaLoadBatch; ++k) {
      const int j = j0 + k * S::kSegs;
      const int64_t g = g0 + j;
      v[k] = live && j < rows && g >= 0 && g < ntime ? ldg_stream(xc + g * ninner) : qnan;
    }
#pragma unroll
    for (int k = 0; k < kPaLoadBatch; ++k) {
      const int j = j0 + k * S::kSegs;
      if (j < rows) xs[j * S::kCells + cl] = v[k];
    }
  }
  __syncthreads();

  // rows 1 .. rows-1 become d[j] = x[j] - x[j-1], from the top down in chunks
  // of kChunk rows: a chunk reads its rows and the one below, then (after the
  // barrier) overwrites only its own rows, which no lower chunk reads.
  constexpr int kChunk = S::kSegs * kPaLoadBatch;
  for (int c0 = ((rows - 1) / kChunk) * kChunk; c0 >= 0; c0 -= kChunk) {
    T d[kPaLoadBatch];
#pragma unroll
    for (int k = 0; k < kPaLoadBatch; ++k) {
      const int j = c0 + sg + k * S::kSegs;
      d[k] = j >= 1 && j < rows ? pa_sub(xs[j * S::kCells + cl], xs[(j - 1) * S::kCells + cl])
                                : qnan;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kPaLoadBatch; ++k) {
      const int j = c0 + sg + k * S::kSegs;
      if (j >= 1 && j < rows) xs[j * S::kCells + cl] = d[k];
    }
  }
  __syncthreads();

  // this thread's outputs a .. a+n-1 (tile rows); output t sums rows t+1 .. t+w
  const int a = sg * S::kSeg;
  const int64_t left = ntime - t0 - a;
  const int n = left < S::kSeg ? int(left) : S::kSeg;
  if (!live || n <= 0) return;
  T* oc = out + (o * ntime + t0) * ninner + cell;
  for (int t = a; t < a + n; t += kPaIlp) {
    double s[kPaIlp];
#pragma unroll
    for (int u = 0; u < kPaIlp; ++u) s[u] = double(xs[(t + u + 1) * S::kCells + cl]);
    for (int k = 2; k <= w; ++k) {
#pragma unroll
      for (int u = 0; u < kPaIlp; ++u)
        s[u] = __dadd_rn(s[u], double(xs[(t + u + k) * S::kCells + cl]));
    }
#pragma unroll
    for (int u = 0; u < kPaIlp; ++u) {
      if (t + u >= a + n) break;
      T r = pa_round(s[u], T());
      if (clamp && r < T(0)) r = T(0);
      oc[int64_t(t + u) * ninner] = r;
    }
  }
}

// Every output NaN: windows of w >= ntime steps, wider than the staged cap.
template <typename T>
__global__ void __launch_bounds__(kPaThreads) precip_nan_kernel(int64_t n, T* __restrict__ out) {
  const T qnan = T(CUDART_NAN);
  for (int64_t i = int64_t(blockIdx.x) * kPaThreads + threadIdx.x; i < n;
       i += int64_t(gridDim.x) * kPaThreads)
    out[i] = qnan;
}

template <typename T>
static size_t pa_smem(int32_t w) {
  return (size_t(kPaBlock) + w) * PaShape<T>::kCells * sizeof(T);
}

static int pa_validate(int dtype, int64_t nouter, int64_t ntime, int64_t ninner,
                       int32_t window) {
  WB2_REQUIRE(dtype == WB2_F32 || dtype == WB2_F64,
              "dtype must be WB2_F32 or WB2_F64 (got %d)", dtype);
  WB2_REQUIRE(nouter >= 0 && ntime >= 0 && ninner >= 0,
              "nouter / ntime / ninner must be >= 0");
  WB2_REQUIRE(window >= 1, "window must be >= 1 (got %d)", window);
  WB2_REQUIRE(window <= kPaMaxWindow || window >= ntime,
              "window = %d is wider than the %d staged steps (and shorter than the series, "
              "ntime = %lld)",
              window, kPaMaxWindow, static_cast<long long>(ntime));
  WB2_REQUIRE((ntime + kPaBlock - 1) / kPaBlock <= 65535,
              "ntime = %lld is too long for the accumulation kernel's grid",
              static_cast<long long>(ntime));
  const int64_t ntile = (ninner + 31) / 32;  // float tiles; double ones are twice as many
  WB2_REQUIRE(nouter * ntile * 2 <= 0x7fffffff,
              "too many cells for the accumulation kernel's grid");
  return WB2_OK;
}

template <typename T>
static int pa_launch(wb2_ctx* ctx, const T* x, int64_t nouter, int64_t ntime, int64_t ninner,
                     int32_t window, int clamp, T* out) {
  if (window >= ntime && window > kPaMaxWindow) {
    const int64_t n = nouter * ntime * ninner;
    const int64_t nblk = std::min<int64_t>((n + kPaThreads - 1) / kPaThreads,
                                           int64_t(ctx->num_sms) * 16);
    precip_nan_kernel<T><<<static_cast<unsigned>(nblk), kPaThreads, 0, ctx->stream>>>(n, out);
  } else {
    constexpr int c = PaShape<T>::kCells;
    const int64_t ntile = (ninner + c - 1) / c;
    const size_t smem = pa_smem<T>(window);
    WB2_CUDA_TRY(cudaFuncSetAttribute(precip_kernel<T>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
    const dim3 grid(static_cast<unsigned>(nouter * ntile),
                    static_cast<unsigned>((ntime + kPaBlock - 1) / kPaBlock));
    precip_kernel<T><<<grid, kPaThreads, smem, ctx->stream>>>(x, ntime, ninner, ntile, window,
                                                             clamp ? 1 : 0, out);
  }
  WB2_CUDA_TRY(cudaGetLastError());
  ctx->launches += 1;
  return WB2_OK;
}

static int pa_launch_any(wb2_ctx* ctx, int dtype, const void* x, int64_t nouter, int64_t ntime,
                         int64_t ninner, int32_t window, int clamp, void* out) {
  if (dtype == WB2_F32)
    return pa_launch(ctx, static_cast<const float*>(x), nouter, ntime, ninner, window, clamp,
                     static_cast<float*>(out));
  return pa_launch(ctx, static_cast<const double*>(x), nouter, ntime, ninner, window, clamp,
                   static_cast<double*>(out));
}

}  // namespace wb2

using namespace wb2;

extern "C" {

int wb2_precip_accumulation(wb2_ctx* ctx, const void* x, int dtype, int64_t nouter,
                            int64_t ntime, int64_t ninner, int32_t window, int clamp_negative,
                            void* out) {
  WB2_NVTX("wb2_precip_accumulation");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_TRY(pa_validate(dtype, nouter, ntime, ninner, window));
  if (nouter == 0 || ntime == 0 || ninner == 0) return WB2_OK;
  WB2_REQUIRE(x != nullptr, "x is NULL");
  WB2_REQUIRE(out != nullptr, "out is NULL");
  DeviceGuard guard(ctx->device);
  return pa_launch_any(ctx, dtype, x, nouter, ntime, ninner, window, clamp_negative, out);
}

int wb2_precip_accumulation_host(wb2_ctx* ctx, const void* x, int dtype, int64_t nouter,
                                 int64_t ntime, int64_t ninner, int32_t window,
                                 int clamp_negative, size_t budget, void* out) {
  WB2_NVTX("wb2_precip_accumulation_host");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_TRY(pa_validate(dtype, nouter, ntime, ninner, window));
  if (nouter == 0 || ntime == 0 || ninner == 0) return WB2_OK;
  WB2_REQUIRE(x != nullptr, "x is NULL");
  WB2_REQUIRE(out != nullptr, "out is NULL");
  DeviceGuard guard(ctx->device);
  char* const out_host[1] = {static_cast<char*>(out)};
  const size_t es = dtype == WB2_F32 ? 4 : 8;
  return stream_series_bands(
      ctx, x, es, es, nouter, ntime, ninner, ntime, false, out_host, 1, budget,
      [&](const void* in, int64_t k, int64_t n, void* const* dev_out) {
        return pa_launch_any(ctx, dtype, in, k, ntime, n, window, clamp_negative, dev_out[0]);
      });
}

}  // extern "C"

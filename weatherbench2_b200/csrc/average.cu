// Means and raw moments over reduced dims: wb2_average (device array) and
// wb2_average_host (NumPy / memmap array streamed in bands).
//
// Replaces the `v * weights` + xbeam.Mean of scripts/compute_averages.py and
// the three xarray means of scripts/compute_statistical_moments.py's
// moment_reduce.  x is read in place in the canonical layout
// [K0][R0][K1][R1][K2]: the K extents are kept, the R extents reduced.  Per
// kept cell (k0, k1, k2), over its n = R0 * R1 samples in the flat order
// s = r0 * R1 + r1, one read of x gives
//   S1 = sum w(s) * x,  S2 = sum w(s) * T(x * x),  N = #non-NaN samples
// from which mean = S1 / count, mean_sq = S2 / count and frac = N / n
// (count = N with skipna, else n).  include/wb2b200.h and DESIGN.md section 8g
// pin the summation order; it depends on n alone:
//   chunk   the samples split into chunks of kAvgChunk consecutive s
//   lane    inside a chunk, sample s goes to class (s mod 32); each class adds
//           its samples in increasing s to a float64 accumulator from +0.0
//   tree    the 32 class sums are added pairwise: c + (c + 16), then + 8, 4,
//           2, 1 (a xor butterfly), giving the chunk's partial
//   chunks  launch_block_sum adds the chunk partials in chunk order from +0.0
// Two kernels map that order to threads; both give the same bits, so the
// choice (from K2 alone) only decides which accesses coalesce:
//   avg_warp_kernel  K2 < 32: one warp per (cell, chunk), lane = class; a
//                    cell's samples are (nearly) contiguous.
//   avg_cell_kernel  K2 >= 32: a CTA per (32 cells, chunk), lane = cell and
//                    warp g holds classes g, g + 8, g + 16, g + 24; the 32
//                    class sums meet in shared memory.
// A cell of one chunk is finalised in the kernel; otherwise each (cell, chunk)
// writes a float64 partial triple, launch_block_sum adds them and
// avg_finalize_kernel divides.  No float atomics: the bits are fixed by the
// shape.
#include <math_constants.h>

#include <algorithm>
#include <type_traits>

#include "region_reduce.cuh"
#include "stage.cuh"

namespace wb2 {

constexpr int64_t kAvgChunk = 65536;  // samples per chunk (a multiple of 32)
constexpr int kAvgThreads = 256;
constexpr int kAvgWarps = kAvgThreads / 32;
constexpr int kAvgCellMin = 32;       // K2 from which the cell kernel is used
constexpr int kAvgStats = 3;          // S1, S2, N
// loads issued before their adds: 8 per lane in the warp kernel, 4 (one per
// accumulator) in the cell kernel, whose 8 would spill
constexpr int kAvgWarpBatch = 8, kAvgCellBatch = 4;

struct AvgShape {
  int64_t K0, R0, K1, R1, K2;
  int64_t n, ncell, nchunk;
};

struct AvgWeights {
  const double* w;  // NULL: unweighted
  int64_t div, len;
};

// The statistics of one call: final outputs (any may be NULL) and, for
// nchunk > 1, the partial triples [ncell][nchunk][3].
struct AvgOut {
  void* mean;
  void* mean_sq;
  double* frac;
  double* partial;
  int skipna;
};

template <typename T, bool kW>
using AvgOutT = typename std::conditional<kW, double, T>::type;

template <typename T>
__device__ __forceinline__ T avg_sq(T v);
template <>
__device__ __forceinline__ float avg_sq(float v) { return __fmul_rn(v, v); }
template <>
__device__ __forceinline__ double avg_sq(double v) { return __dmul_rn(v, v); }

__device__ __forceinline__ float avg_round(double v, float*) { return __double2float_rn(v); }
__device__ __forceinline__ double avg_round(double v, double*) { return v; }

// Adds the samples s, s + step, ... (< s_end) of the cell whose first sample is
// at `xc` into the accumulators, the i-th of them into a[i % kAcc] (kAcc
// divides kBatch).  (r0, r1)
// and the weight index follow s as mixed-radix counters, so the loop divides
// nothing.
template <typename T, bool kW, int kAcc, int kBatch>
__device__ __forceinline__ void avg_accumulate(const T* __restrict__ xc, const AvgShape& sh,
                                               const AvgWeights& wt, int skipna, int64_t s,
                                               int64_t s_end, int step, double (&a1)[kAcc],
                                               double (&a2)[kAcc], int (&cnt)[kAcc]) {
  const int64_t st0 = sh.K1 * sh.R1 * sh.K2;
  int64_t r0 = s / sh.R1, r1 = s - r0 * sh.R1;
  const int64_t dq = step / sh.R1, dr = step - dq * sh.R1;
  int64_t wq = 0, wr = 0, dwq = 0, dwr = 0;
  if (kW) {
    const int64_t q = s / wt.div, sq = step / wt.div;
    wr = s - q * wt.div;
    wq = q % wt.len;
    dwr = step - sq * wt.div;
    dwq = sq % wt.len;
  }
  const bool skip = skipna != 0;
  while (s < s_end) {
    // kBatch loads in flight before the first add; the adds then follow
    // in sample order, so the bits are those of one load at a time
    T v[kBatch];
    double w[kBatch];
    bool ok[kBatch];
#pragma unroll
    for (int k = 0; k < kBatch; ++k) {
      ok[k] = s < s_end;
      v[k] = T(0);
      w[k] = 1.0;
      if (ok[k]) {
        v[k] = __ldg(xc + r0 * st0 + r1 * sh.K2);
        if (kW) w[k] = __ldg(wt.w + wq);
        s += step;
        r1 += dr;
        r0 += dq;
        if (r1 >= sh.R1) {
          r1 -= sh.R1;
          ++r0;
        }
        if (kW) {
          wr += dwr;
          wq += dwq;
          if (wr >= wt.div) {
            wr -= wt.div;
            ++wq;
          }
          if (wq >= wt.len) wq -= wt.len;
        }
      }
    }
#pragma unroll
    for (int k = 0; k < kBatch; ++k) {
      if (ok[k]) {
        const int a = k % kAcc;
        const bool nan = v[k] != v[k];
        double y = double(v[k]), z = double(avg_sq(v[k]));
        if (kW) {
          y = __dmul_rn(y, w[k]);
          z = __dmul_rn(z, w[k]);
        }
        // adding +0.0 leaves an accumulator unchanged: it starts at +0.0 and
        // so is never -0.0
        a1[a] = __dadd_rn(a1[a], skip && nan ? 0.0 : y);
        a2[a] = __dadd_rn(a2[a], skip && nan ? 0.0 : z);
        cnt[a] += !nan;
      }
    }
  }
}

// Element offset of cell c's first sample.
__device__ __forceinline__ int64_t avg_cell_base(const AvgShape& sh, int64_t c) {
  const int64_t t = c / sh.K2, k2 = c - t * sh.K2;
  const int64_t k0 = t / sh.K1, k1 = t - k0 * sh.K1;
  return ((k0 * sh.R0 * sh.K1 + k1) * sh.R1) * sh.K2 + k2;
}

// Writes cell c's outputs from its sums.
template <typename T, bool kW>
__device__ __forceinline__ void avg_store(const AvgOut& o, int64_t n, int64_t c, double s1,
                                          double s2, double cnt) {
  using O = AvgOutT<T, kW>;
  const double div = o.skipna ? cnt : double(n);
  if (o.mean) static_cast<O*>(o.mean)[c] = avg_round(__ddiv_rn(s1, div), (O*)nullptr);
  if (o.mean_sq) static_cast<O*>(o.mean_sq)[c] = avg_round(__ddiv_rn(s2, div), (O*)nullptr);
  if (o.frac) o.frac[c] = __ddiv_rn(cnt, double(n));
}

template <typename T, bool kW>
__device__ __forceinline__ void avg_emit(const AvgShape& sh, const AvgOut& o, int64_t cell,
                                         int64_t ch, double s1, double s2, double cnt) {
  if (sh.nchunk == 1) {
    avg_store<T, kW>(o, sh.n, cell, s1, s2, cnt);
  } else {
    double* p = o.partial + (cell * sh.nchunk + ch) * kAvgStats;
    p[0] = s1;
    p[1] = s2;
    p[2] = cnt;
  }
}

template <typename T, bool kW>
__global__ void __launch_bounds__(kAvgThreads)
    avg_warp_kernel(const T* __restrict__ x, const AvgShape sh, const AvgWeights wt,
                    const AvgOut o) {
  const int lane = threadIdx.x & 31;
  const int64_t item = int64_t(blockIdx.x) * kAvgWarps + (threadIdx.x >> 5);
  if (item >= sh.ncell * sh.nchunk) return;
  const int64_t cell = item / sh.nchunk, ch = item - cell * sh.nchunk;
  const int64_t s0 = ch * kAvgChunk;
  double a1[1] = {0.0}, a2[1] = {0.0};
  int cnt[1] = {0};
  avg_accumulate<T, kW, 1, kAvgWarpBatch>(x + avg_cell_base(sh, cell), sh, wt, o.skipna, s0 + lane,
                           std::min(sh.n, s0 + kAvgChunk), 32, a1, a2, cnt);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    a1[0] = __dadd_rn(a1[0], __shfl_xor_sync(0xffffffffu, a1[0], off));
    a2[0] = __dadd_rn(a2[0], __shfl_xor_sync(0xffffffffu, a2[0], off));
    cnt[0] += __shfl_xor_sync(0xffffffffu, cnt[0], off);
  }
  if (lane == 0) avg_emit<T, kW>(sh, o, cell, ch, a1[0], a2[0], double(cnt[0]));
}

template <typename T, bool kW>
__global__ void __launch_bounds__(kAvgThreads)
    avg_cell_kernel(const T* __restrict__ x, const AvgShape sh, const AvgWeights wt,
                    const AvgOut o) {
  __shared__ double t1[32][33], t2[32][33];
  __shared__ int tc[32][33];
  const int j = threadIdx.x & 31, g = threadIdx.x >> 5;
  const int64_t cb = blockIdx.x / sh.nchunk, ch = blockIdx.x - cb * sh.nchunk;
  const int64_t cell = cb * 32 + j;
  double a1[4] = {0.0, 0.0, 0.0, 0.0}, a2[4] = {0.0, 0.0, 0.0, 0.0};
  int cnt[4] = {0, 0, 0, 0};
  if (cell < sh.ncell) {
    const int64_t s0 = ch * kAvgChunk;
    // warp g's i-th sample is s0 + g + 8 i, of class g + 8 (i mod 4)
    avg_accumulate<T, kW, 4, kAvgCellBatch>(x + avg_cell_base(sh, cell), sh, wt, o.skipna, s0 + g,
                             std::min(sh.n, s0 + kAvgChunk), kAvgWarps, a1, a2, cnt);
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    t1[g + 8 * k][j] = a1[k];
    t2[g + 8 * k][j] = a2[k];
    tc[g + 8 * k][j] = cnt[k];
  }
  __syncthreads();
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    for (int e = threadIdx.x; e < off * 32; e += kAvgThreads) {
      const int l = e >> 5, c = e & 31;
      t1[l][c] = __dadd_rn(t1[l][c], t1[l + off][c]);
      t2[l][c] = __dadd_rn(t2[l][c], t2[l + off][c]);
      tc[l][c] += tc[l + off][c];
    }
    __syncthreads();
  }
  if (g == 0 && cell < sh.ncell)
    avg_emit<T, kW>(sh, o, cell, ch, t1[0][j], t2[0][j], double(tc[0][j]));
}

template <typename T, bool kW>
__global__ void avg_finalize_kernel(const double* __restrict__ sums, int64_t n, int64_t ncell,
                                    const AvgOut o) {
  const int64_t c = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (c >= ncell) return;
  const double* p = sums + c * kAvgStats;
  avg_store<T, kW>(o, n, c, p[0], p[1], p[2]);
}

// ---- launch ------------------------------------------------------------------
static int64_t avg_nchunk(int64_t n) { return (n + kAvgChunk - 1) / kAvgChunk; }

// Device bytes of the partial triples and their sums for `ncell` cells.
static size_t avg_scratch_bytes(int64_t ncell, int64_t n) {
  const int64_t nchunk = avg_nchunk(n);
  return nchunk > 1 ? size_t(ncell) * (nchunk + 1) * kAvgStats * sizeof(double) : 0;
}

template <typename T, bool kW>
static int avg_launch_t(wb2_ctx* ctx, const T* x, const AvgShape& sh, const AvgWeights& wt,
                        AvgOut o, double* scratch) {
  double* sums = nullptr;
  if (sh.nchunk > 1) {
    o.partial = scratch;
    sums = scratch + sh.ncell * sh.nchunk * kAvgStats;
  }
  if (sh.K2 >= kAvgCellMin) {
    const int64_t blocks = (sh.ncell + 31) / 32 * sh.nchunk;
    WB2_TRY(launch_kernel(ctx, avg_cell_kernel<T, kW>, dim3(static_cast<unsigned>(blocks)),
                          kAvgThreads, 0, x, sh, wt, o));
  } else {
    const int64_t blocks = (sh.ncell * sh.nchunk + kAvgWarps - 1) / kAvgWarps;
    WB2_TRY(launch_kernel(ctx, avg_warp_kernel<T, kW>, dim3(static_cast<unsigned>(blocks)),
                          kAvgThreads, 0, x, sh, wt, o));
  }
  ctx->launches += 1;
  if (sh.nchunk > 1) {
    WB2_TRY(launch_block_sum(ctx, o.partial, sums, sh.ncell, int(sh.nchunk), kAvgStats));
    WB2_TRY(launch_kernel(ctx, avg_finalize_kernel<T, kW>,
                          dim3(static_cast<unsigned>((sh.ncell + 255) / 256)), 256, 0,
                          static_cast<const double*>(sums), sh.n, sh.ncell, o));
    ctx->launches += 2;
  }
  return WB2_OK;
}

static int avg_launch(wb2_ctx* ctx, int dtype, const void* x, const AvgShape& sh,
                      const AvgWeights& wt, const AvgOut& o, double* scratch) {
  if (dtype == WB2_F32)
    return wt.w ? avg_launch_t<float, true>(ctx, static_cast<const float*>(x), sh, wt, o, scratch)
                : avg_launch_t<float, false>(ctx, static_cast<const float*>(x), sh, wt, o, scratch);
  return wt.w ? avg_launch_t<double, true>(ctx, static_cast<const double*>(x), sh, wt, o, scratch)
              : avg_launch_t<double, false>(ctx, static_cast<const double*>(x), sh, wt, o, scratch);
}

static AvgShape avg_shape(int64_t k0, int64_t r0, int64_t k1, int64_t r1, int64_t k2) {
  AvgShape sh{k0, r0, k1, r1, k2, r0 * r1, k0 * k1 * k2, 0};
  sh.nchunk = avg_nchunk(sh.n);
  return sh;
}

static int avg_validate(int dtype, const AvgShape& sh, const double* weights, int64_t wdiv,
                        int64_t wlen, const void* mean, const void* mean_sq, const double* frac) {
  WB2_REQUIRE(dtype == WB2_F32 || dtype == WB2_F64,
              "dtype must be WB2_F32 or WB2_F64 (got %d)", dtype);
  WB2_REQUIRE(sh.R0 >= 1 && sh.R1 >= 1, "reduced extents r0 and r1 must be >= 1 (got %lld, %lld)",
              static_cast<long long>(sh.R0), static_cast<long long>(sh.R1));
  WB2_REQUIRE(sh.K0 >= 0 && sh.K1 >= 0 && sh.K2 >= 0, "kept extents k0, k1 and k2 must be >= 0");
  if (weights)
    WB2_REQUIRE(wdiv >= 1 && wlen >= 1 && sh.n % wdiv == 0 && (sh.n / wdiv) % wlen == 0,
                "weights (wdiv %lld, wlen %lld) do not fit the sample index of %lld samples",
                static_cast<long long>(wdiv), static_cast<long long>(wlen),
                static_cast<long long>(sh.n));
  WB2_REQUIRE(mean || mean_sq || frac, "no output requested: mean, mean_sq and frac are NULL");
  WB2_REQUIRE(sh.ncell == 0 || sh.nchunk <= 0x7fffffff / kAvgStats,
              "too many samples per cell for the average kernels");
  WB2_REQUIRE(sh.ncell == 0 || sh.ncell <= (int64_t(0x7fffffff) * kAvgWarps) / sh.nchunk,
              "too many cells x chunks for the average kernels' grid");
  return WB2_OK;
}

// The weight table in device memory held by `blk`.
static int avg_weights(wb2_ctx* ctx, const double* weights, int64_t wdiv, int64_t wlen,
                       DeviceBlock* blk, AvgWeights* wt) {
  *wt = AvgWeights{nullptr, wdiv, wlen};
  if (!weights) return WB2_OK;
  size_t off[1];
  WB2_TRY(upload_parts(ctx, {{weights, size_t(wlen) * sizeof(double)}}, blk, off));
  wt->w = blk->at<double>(off[0]);
  return WB2_OK;
}

}  // namespace wb2

using namespace wb2;

extern "C" {

int wb2_average(wb2_ctx* ctx, const void* x, int dtype, int64_t k0, int64_t r0, int64_t k1,
                int64_t r1, int64_t k2, const double* weights, int64_t wdiv, int64_t wlen,
                int skipna, void* mean, void* mean_sq, double* frac) {
  WB2_NVTX("wb2_average");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  const AvgShape sh = avg_shape(k0, r0, k1, r1, k2);
  WB2_TRY(avg_validate(dtype, sh, weights, wdiv, wlen, mean, mean_sq, frac));
  if (sh.ncell == 0) return WB2_OK;
  WB2_REQUIRE(x != nullptr, "x is NULL");
  DeviceGuard guard(ctx->device);
  DeviceBlock wblk, scratch;
  AvgWeights wt;
  WB2_TRY(avg_weights(ctx, weights, wdiv, wlen, &wblk, &wt));
  const size_t sb = avg_scratch_bytes(sh.ncell, sh.n);
  if (sb) WB2_TRY(scratch.alloc(ctx, sb));
  return avg_launch(ctx, dtype, x, sh, wt, AvgOut{mean, mean_sq, frac, nullptr, skipna ? 1 : 0},
                    sb ? scratch.at<double>(0) : nullptr);
}

// A band holds whole cells, so it adds the same numbers in the same order as
// the device entry: k2 cells [R0][R1][nb] of one (k0, k1) when a k1 slice does
// not fit (one 3-D copy), else k1 slices [R0][m][R1][K2] of one k0 (one 2-D
// copy of R0 rows), else whole k0 slabs.
int wb2_average_host(wb2_ctx* ctx, const void* x, int dtype, int64_t k0, int64_t r0, int64_t k1,
                     int64_t r1, int64_t k2, const double* weights, int64_t wdiv, int64_t wlen,
                     int skipna, size_t budget, void* mean, void* mean_sq, double* frac) {
  WB2_NVTX("wb2_average_host");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  const AvgShape sh = avg_shape(k0, r0, k1, r1, k2);
  WB2_TRY(avg_validate(dtype, sh, weights, wdiv, wlen, mean, mean_sq, frac));
  if (sh.ncell == 0) return WB2_OK;
  WB2_REQUIRE(x != nullptr, "x is NULL");
  DeviceGuard guard(ctx->device);
  const size_t es = dtype == WB2_F32 ? 4 : 8;
  const size_t mes = weights ? 8 : es;
  char* const out_host[3] = {static_cast<char*>(mean), static_cast<char*>(mean_sq),
                             reinterpret_cast<char*>(frac)};
  const size_t out_es[3] = {mes, mes, 8};
  size_t cell_out = 0;
  for (int s = 0; s < 3; ++s) cell_out += out_host[s] ? out_es[s] : 0;
  // device bytes per cell: its samples and outputs in both buffers, plus its
  // chunk partials
  const size_t cell_in = size_t(sh.n) * es;
  const size_t cell_cost = 2 * (cell_in + cell_out) + avg_scratch_bytes(1, sh.n);
  const int64_t ncb = static_cast<int64_t>(budget / cell_cost);
  WB2_REQUIRE(ncb >= 1,
              "budget of %zu bytes is below the %zu device bytes one cell (r0 x r1 = %lld "
              "samples) needs",
              budget, cell_cost, static_cast<long long>(sh.n));
  const int64_t nb = std::min(ncb, sh.K2);
  const int64_t nk1 = nb == sh.K2 ? std::max<int64_t>(1, std::min(ncb / sh.K2, sh.K1)) : 1;
  const int64_t ko = nb == sh.K2 && nk1 == sh.K1
                         ? std::max<int64_t>(1, std::min(ncb / (sh.K1 * sh.K2), sh.K0))
                         : 1;
  const int64_t band_cells = ko * nk1 * nb;
  auto al = [](size_t b) { return (b + 255) / 256 * 256; };
  const size_t b_in = al(size_t(band_cells) * cell_in);
  size_t b_out[3];
  size_t stage_bytes = b_in;
  for (int s = 0; s < 3; ++s) {
    b_out[s] = out_host[s] ? al(size_t(band_cells) * out_es[s]) : 0;
    stage_bytes += b_out[s];
  }

  DeviceBlock wblk, scratch;
  AvgWeights wt;
  WB2_TRY(avg_weights(ctx, weights, wdiv, wlen, &wblk, &wt));
  const size_t sb = avg_scratch_bytes(band_cells, sh.n);
  if (sb) WB2_TRY(scratch.alloc(ctx, sb));
  StagePair stage;
  WB2_TRY(stage.alloc(stage_bytes));
  StagePipe pipe(ctx, stage.buf[0], stage.buf[1]);
  const char* xh = static_cast<const char*>(x);
  const size_t row = size_t(sh.K1) * sh.R1 * sh.K2 * es;  // one r0 row of one k0
  for (int64_t o0 = 0; o0 < sh.K0; o0 += ko) {
    const int64_t kb = std::min(ko, sh.K0 - o0);
    for (int64_t a = 0; a < sh.K1; a += nk1) {
      const int64_t m = std::min(nk1, sh.K1 - a);
      for (int64_t c0 = 0; c0 < sh.K2; c0 += nb) {
        const int64_t nc = std::min(nb, sh.K2 - c0);
        char* in;
        WB2_TRY(pipe.next(&in));
        void* out[3] = {nullptr, nullptr, nullptr};
        char* op = in + b_in;
        for (int s = 0; s < 3; ++s)
          if (out_host[s]) {
            out[s] = op;
            op += b_out[s];
          }
        const char* src = xh + size_t(o0) * sh.R0 * row + (size_t(a) * sh.R1 * sh.K2 + c0) * es;
        AvgShape band;
        if (nb < sh.K2) {  // [R0][R1][nc]: R1 rows K2 apart in each of R0 planes
          WB2_TRY(pipe.h2d_3d(in, src, size_t(sh.K2) * es, size_t(sh.K1) * sh.R1,
                              size_t(nc) * es, size_t(sh.R1), size_t(sh.R0)));
          band = avg_shape(1, sh.R0, 1, sh.R1, nc);
        } else {
          const size_t width = size_t(m) * sh.R1 * sh.K2 * es;
          WB2_TRY(pipe.h2d_2d(in, width, src, row, width, size_t(kb) * sh.R0));
          band = avg_shape(kb, sh.R0, m, sh.R1, sh.K2);
        }
        WB2_TRY(pipe.ready());
        WB2_TRY(avg_launch(ctx, dtype, in, band, wt,
                           AvgOut{out[0], out[1], static_cast<double*>(out[2]), nullptr,
                                  skipna ? 1 : 0},
                           sb ? scratch.at<double>(0) : nullptr));
        const size_t first = (size_t(o0) * sh.K1 + a) * sh.K2 + c0;
        for (int s = 0; s < 3; ++s)
          if (out_host[s])
            WB2_TRY(pipe.d2h(out_host[s] + first * out_es[s], out[s],
                             size_t(band.ncell) * out_es[s]));
        WB2_TRY(pipe.done());
      }
    }
  }
  return pipe.finish();
}

}  // extern "C"

// Column integrals over the pressure-level axis (sm_90a): total column water,
// integrated water transport and eddy kinetic energy of
// weatherbench2/derived_variables.py:212-228 and 365-430, one kernel per kind.
//
// All three end in xarray's integrate('level'), i.e. duck_array_ops.trapz:
//   sum(dx * 0.5 * (y[1:] + y[:-1]), skipna=False),  dx = level[1:] - level[:-1]
// With T the data type, the pair sum y[k] + y[k+1] is a T addition and the rest
// is float64.  The host passes w_k = 0.5 * (level[k+1] - level[k]) in float64,
// and every kernel forms S = w_0 p_0 + w_1 p_1 + ... in float64 from k = 0
// upward, starting from the k = 0 term, with correctly rounded intrinsics only,
// so nothing is contracted into an FMA:
//   total column  (1 / 9.81) * S(q)
//   IVT           (1 / 9.81) * sqrt(S(q*u)^2 + S(q*v)^2), q*u rounded in T
//   EKE           0.5 * S(u'^2 + v'^2), u' = u - zonal NaN-skipping mean, float64
// and the result is rounded once to T.
//
// Total column and IVT: one thread per output cell walks the levels of
// [nouter][nlev][ninner]; consecutive threads read consecutive inner cells.
// EKE in the [nrow][nlon] layout: one CTA per (outer, row) stages each level's
// row of u and v in shared memory while it reduces the zonal mean, so HBM sees
// one read of every input and one write of the output.  EKE in the [nlon][nrow]
// layout: eke_tile_kernel below, whose warps read adjacent rows.
#include <algorithm>

#include "common.cuh"

namespace wb2 {
namespace {

constexpr double kInvG = 1 / 9.81;  // `1 / g * x` in derived_variables.py:385, 430
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ void store(float* p, double x) { *p = __double2float_rn(x); }
__device__ __forceinline__ void store(double* p, double x) { *p = x; }

// adds the term of level pair (k-1, k) to the running sum s
__device__ __forceinline__ void add_term(double& s, int k, double term) {
  s = k == 1 ? term : __dadd_rn(s, term);
}

template <typename T, bool kIvt>
__global__ void __launch_bounds__(kThreads)
    column_kernel(const T* __restrict__ q, const T* __restrict__ u, const T* __restrict__ v,
                  int64_t nouter, int64_t outer_stride, int32_t nlev, int64_t ninner,
                  const double* __restrict__ w, T* __restrict__ out) {
  const int64_t n = nouter * ninner;
  for (int64_t cell = int64_t(blockIdx.x) * kThreads + threadIdx.x; cell < n;
       cell += int64_t(gridDim.x) * kThreads) {
    const int64_t o = cell / ninner;
    int64_t at = o * outer_stride + (cell - o * ninner);
    double su = 0.0, sv = 0.0;
    if (nlev > 0) {
      T qk = ldg_stream(q + at);
      T yu = kIvt ? mul_rn(qk, ldg_stream(u + at)) : qk;
      T yv = kIvt ? mul_rn(qk, ldg_stream(v + at)) : T(0);
#pragma unroll 4
      for (int k = 1; k < nlev; ++k) {
        at += ninner;
        const double wk = __ldg(w + k - 1);
        qk = ldg_stream(q + at);
        const T cu = kIvt ? mul_rn(qk, ldg_stream(u + at)) : qk;
        add_term(su, k, __dmul_rn(wk, double(add_rn(yu, cu))));
        yu = cu;
        if constexpr (kIvt) {
          const T cv = mul_rn(qk, ldg_stream(v + at));
          add_term(sv, k, __dmul_rn(wk, double(add_rn(yv, cv))));
          yv = cv;
        }
      }
    }
    double r;
    if constexpr (kIvt)
      r = __dmul_rn(kInvG, __dsqrt_rn(__dadd_rn(__dmul_rn(su, su), __dmul_rn(sv, sv))));
    else
      r = __dmul_rn(kInvG, su);
    store(out + cell, r);
  }
}

// Sums a per-thread (sum, count) over the CTA in a fixed order: a shuffle tree
// per warp, then the warp partials in warp order.  `part` is this level's
// buffer; the caller alternates two so one barrier per level suffices.
__device__ __forceinline__ double cta_mean(double s, int c, double* part_s, int* part_c) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    s = __dadd_rn(s, __shfl_down_sync(0xffffffffu, s, off));
    c += __shfl_down_sync(0xffffffffu, c, off);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) {
    part_s[warp] = s;
    part_c[warp] = c;
  }
  __syncthreads();
  double ts = part_s[0];
  int tc = part_c[0];
#pragma unroll
  for (int i = 1; i < kWarps; ++i) {
    ts = __dadd_rn(ts, part_s[i]);
    tc += part_c[i];
  }
  return __ddiv_rn(ts, double(tc));  // 0 / 0 = NaN for an all-NaN row
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
    eke_kernel(const T* __restrict__ u, const T* __restrict__ v, int32_t nrow, int32_t nlon,
               int64_t row_stride, int64_t lon_stride, int64_t outer_stride, int32_t nlev,
               int64_t ninner, const double* __restrict__ w, T* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char smem[];
  double* prev = reinterpret_cast<double*>(smem);  // [nlon] y of the previous level
  double* acc = prev + nlon;                       // [nlon] running level sum
  T* us = reinterpret_cast<T*>(acc + nlon);        // [nlon] this level's row of u
  T* vs = us + nlon;                               // [nlon] and of v
  __shared__ double part_s[2][2][kWarps];
  __shared__ int part_c[2][2][kWarps];
  const int64_t o = blockIdx.x / nrow;
  const int32_t row = static_cast<int32_t>(blockIdx.x - o * nrow);
  const int64_t base = o * outer_stride + row * row_stride;
  // cell c belongs to thread c % kThreads in every loop, so the per-cell
  // arrays need no barrier
  for (int k = 0; k < nlev; ++k) {
    const T* uk = u + base + k * ninner;
    const T* vk = v + base + k * ninner;
    double su = 0.0, sv = 0.0;
    int nu = 0, nv = 0;
    for (int c = threadIdx.x; c < nlon; c += kThreads) {
      const T a = ldg_stream(uk + c * lon_stride), b = ldg_stream(vk + c * lon_stride);
      us[c] = a;
      vs[c] = b;
      if (a == a) {  // xarray's mean skips NaN
        su = __dadd_rn(su, double(a));
        ++nu;
      }
      if (b == b) {
        sv = __dadd_rn(sv, double(b));
        ++nv;
      }
    }
    const double mu = cta_mean(su, nu, part_s[k & 1][0], part_c[k & 1][0]);
    const double mv = cta_mean(sv, nv, part_s[k & 1][1], part_c[k & 1][1]);
    const double wk = k > 0 ? __ldg(w + k - 1) : 0.0;
    for (int c = threadIdx.x; c < nlon; c += kThreads) {
      const double du = __dsub_rn(double(us[c]), mu), dv = __dsub_rn(double(vs[c]), mv);
      const double y = __dadd_rn(__dmul_rn(du, du), __dmul_rn(dv, dv));
      if (k > 0) {
        const double term = __dmul_rn(wk, __dadd_rn(prev[c], y));
        acc[c] = k == 1 ? term : __dadd_rn(acc[c], term);
      }
      prev[c] = y;
    }
  }
  T* ob = out + o * ninner + row * row_stride;
  for (int c = threadIdx.x; c < nlon; c += kThreads)
    store(ob + c * lon_stride, nlev > 1 ? __dmul_rn(0.5, acc[c]) : 0.0);
}

// EKE in the [nlon][nrow] layout, where adjacent rows are adjacent in memory:
// a CTA owns `tile` adjacent rows (a power of 2, at most 8) and thread t
// handles row t % tile at longitudes t / tile + m * (kTileThreads / tile), so
// a warp reads 32 / tile longitudes of `tile` consecutive cells each.  Per
// level, the first pass sums each row, the partials are reduced in a fixed
// order (shuffles over the lanes of a row, then the warps in order), and the
// second pass re-reads the tile's cells -- tile * nlon * 2 values, which L2
// still holds -- to form the anomalies.  The per-cell running sums of all
// levels stay in shared memory ([nlon][tile] doubles, twice).
constexpr int kTileThreads = 1024;
constexpr int kTileWarps = kTileThreads / 32;
constexpr int kMaxTile = 8;

template <typename T>
__global__ void __launch_bounds__(kTileThreads)
    eke_tile_kernel(const T* __restrict__ u, const T* __restrict__ v, int32_t nrow,
                    int32_t nlon, int32_t tile, int64_t outer_stride, int32_t nlev,
                    int64_t ninner, const double* __restrict__ w, T* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char smem[];
  double* prev = reinterpret_cast<double*>(smem);  // [nlon][tile] y of the previous level
  double* acc = prev + size_t(nlon) * tile;        // [nlon][tile] running level sum
  __shared__ double part_s[2][2][kTileWarps][kMaxTile];
  __shared__ int part_c[2][2][kTileWarps][kMaxTile];
  const int32_t ntile = (nrow + tile - 1) / tile;
  const int64_t o = blockIdx.x / ntile;
  const int32_t row0 = static_cast<int32_t>(blockIdx.x - o * ntile) * tile;
  const int r = threadIdx.x & (tile - 1);
  const int j0 = threadIdx.x / tile, jstep = kTileThreads / tile;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool live = row0 + r < nrow;
  const int64_t base = o * outer_stride + row0 + r;
  for (int k = 0; k < nlev; ++k) {
    const T* uk = u + base + k * ninner;
    const T* vk = v + base + k * ninner;
    double su = 0.0, sv = 0.0;
    int nu = 0, nv = 0;
    if (live) {
      // branch-free so that the loads of several longitudes are in flight at
      // once; adding +0 for a NaN cell leaves the sum as it is (it is never -0)
#pragma unroll 4
      for (int c = j0; c < nlon; c += jstep) {
        const T a = __ldg(uk + int64_t(c) * nrow), b = __ldg(vk + int64_t(c) * nrow);
        su = __dadd_rn(su, a == a ? double(a) : 0.0);  // xarray's mean skips NaN
        sv = __dadd_rn(sv, b == b ? double(b) : 0.0);
        nu += a == a;
        nv += b == b;
      }
    }
    // lanes r, r + tile, r + 2 tile, ... of a warp hold the same row
    for (int off = 16; off >= tile; off >>= 1) {
      su = __dadd_rn(su, __shfl_down_sync(0xffffffffu, su, off));
      sv = __dadd_rn(sv, __shfl_down_sync(0xffffffffu, sv, off));
      nu += __shfl_down_sync(0xffffffffu, nu, off);
      nv += __shfl_down_sync(0xffffffffu, nv, off);
    }
    double(*ps)[kTileWarps][kMaxTile] = part_s[k & 1];
    int(*pc)[kTileWarps][kMaxTile] = part_c[k & 1];
    if (lane < tile) {
      ps[0][warp][lane] = su;
      ps[1][warp][lane] = sv;
      pc[0][warp][lane] = nu;
      pc[1][warp][lane] = nv;
    }
    __syncthreads();
    double tu = ps[0][0][r], tv = ps[1][0][r];
    int cu = pc[0][0][r], cv = pc[1][0][r];
#pragma unroll
    for (int i = 1; i < kTileWarps; ++i) {
      tu = __dadd_rn(tu, ps[0][i][r]);
      tv = __dadd_rn(tv, ps[1][i][r]);
      cu += pc[0][i][r];
      cv += pc[1][i][r];
    }
    const double mu = __ddiv_rn(tu, double(cu)), mv = __ddiv_rn(tv, double(cv));
    const double wk = k > 0 ? __ldg(w + k - 1) : 0.0;
    if (live) {
#pragma unroll 4
      for (int c = j0; c < nlon; c += jstep) {
        const double du = __dsub_rn(double(__ldg(uk + int64_t(c) * nrow)), mu);
        const double dv = __dsub_rn(double(__ldg(vk + int64_t(c) * nrow)), mv);
        const double y = __dadd_rn(__dmul_rn(du, du), __dmul_rn(dv, dv));
        const int at = c * tile + r;
        if (k > 0) {
          const double term = __dmul_rn(wk, __dadd_rn(prev[at], y));
          acc[at] = k == 1 ? term : __dadd_rn(acc[at], term);
        }
        prev[at] = y;
      }
    }
  }
  if (!live) return;
  T* ob = out + o * ninner + row0 + r;
  for (int c = j0; c < nlon; c += jstep)
    store(ob + int64_t(c) * nrow, nlev > 1 ? __dmul_rn(0.5, acc[c * tile + r]) : 0.0);
}

// Rows per CTA of eke_tile_kernel: the largest power of 2 up to kMaxTile whose
// running sums fit in shared memory (0: not even one row fits).
int eke_tile(int32_t nlon, int max_smem) {
  int tile = kMaxTile;
  while (tile > 0 && size_t(tile) * nlon * 16 + 16384 > size_t(max_smem)) tile /= 2;
  return tile;
}

template <typename T>
int launch(wb2_ctx* ctx, int kind, const T* q, const T* u, const T* v, int64_t nouter,
           int64_t outer_stride, int32_t nlev, int64_t ninner, int32_t nlon, int64_t lon_stride,
           int tile, const double* w, T* out) {
  const int32_t nrow = kind == WB2_COL_EKE ? static_cast<int32_t>(ninner / nlon) : 0;
  if (kind == WB2_COL_EKE && lon_stride == 1) {  // [nrow][nlon]
    const size_t smem = size_t(nlon) * (2 * sizeof(double) + 2 * sizeof(T));
    WB2_TRY(launch_kernel(ctx, eke_kernel<T>, dim3(static_cast<unsigned>(nouter * nrow)),
                          kThreads, smem, u, v, nrow, nlon, int64_t(nlon), lon_stride,
                          outer_stride, nlev, ninner, w, out));
  } else if (kind == WB2_COL_EKE) {  // [nlon][nrow]
    const int32_t ntile = (nrow + tile - 1) / tile;
    const size_t smem = size_t(tile) * nlon * 2 * sizeof(double);
    WB2_TRY(launch_kernel(ctx, eke_tile_kernel<T>, dim3(static_cast<unsigned>(nouter * ntile)),
                          kTileThreads, smem, u, v, nrow, nlon, tile, outer_stride, nlev,
                          ninner, w, out));
  } else {
    const int64_t nblk = std::min<int64_t>((nouter * ninner + kThreads - 1) / kThreads,
                                           int64_t(ctx->num_sms) * 16);
    auto kernel = kind == WB2_COL_IVT ? column_kernel<T, true> : column_kernel<T, false>;
    WB2_TRY(launch_kernel(ctx, kernel, dim3(static_cast<unsigned>(nblk)), kThreads, 0, q, u, v,
                          nouter, outer_stride, nlev, ninner, w, out));
  }
  ctx->launches += 1;
  return WB2_OK;
}

}  // namespace
}  // namespace wb2

using namespace wb2;

extern "C" int wb2_column_integral(wb2_ctx* ctx, int kind, int dtype, const void* q,
                                   const void* u, const void* v, int64_t nouter,
                                   int64_t outer_stride, int32_t nlev, int64_t ninner,
                                   int32_t nlon, int64_t lon_stride, const double* weight,
                                   void* out) {
  WB2_NVTX("wb2_column_integral");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_REQUIRE(kind >= WB2_COL_TOTAL_COLUMN && kind <= WB2_COL_EKE,
              "wb2_column_integral: unknown kind %d", kind);
  WB2_REQUIRE(dtype == WB2_F32 || dtype == WB2_F64, "wb2_column_integral: unknown dtype %d",
              dtype);
  WB2_REQUIRE(nouter >= 0 && nlev >= 0 && ninner >= 0, "wb2_column_integral: negative size");
  WB2_REQUIRE(outer_stride >= int64_t(nlev) * ninner,
              "wb2_column_integral: outer_stride %lld is below nlev * ninner = %lld",
              static_cast<long long>(outer_stride), static_cast<long long>(int64_t(nlev) * ninner));
  const int32_t nrow = kind == WB2_COL_EKE && nlon > 0 ? static_cast<int32_t>(ninner / nlon) : 0;
  if (kind == WB2_COL_EKE) {
    WB2_REQUIRE(nlon > 0 && ninner % nlon == 0 && ninner / nlon <= INT32_MAX,
                "wb2_column_integral: ninner = %lld is not a whole number of rows of nlon = %d",
                static_cast<long long>(ninner), nlon);
    WB2_REQUIRE(lon_stride == 1 || lon_stride == nrow,
                "wb2_column_integral: lon_stride %lld is neither 1 nor nrow = %d",
                static_cast<long long>(lon_stride), nrow);
    WB2_REQUIRE(nouter * nrow <= INT32_MAX, "wb2_column_integral: too many rows for the grid");
  }
  WB2_REQUIRE(out != nullptr, "wb2_column_integral: NULL out");
  WB2_REQUIRE(kind == WB2_COL_EKE || q != nullptr, "wb2_column_integral: NULL q");
  WB2_REQUIRE(kind == WB2_COL_TOTAL_COLUMN || (u != nullptr && v != nullptr),
              "wb2_column_integral: NULL u or v");
  WB2_REQUIRE(nlev < 2 || weight != nullptr, "wb2_column_integral: NULL weight");
  if (nouter == 0 || ninner == 0) return WB2_OK;
  DeviceGuard guard(ctx->device);
  int tile = 0;
  if (kind == WB2_COL_EKE) {
    int max_smem = 0;
    WB2_CUDA_TRY(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin,
                                        ctx->device));
    const size_t row_bytes =
        size_t(nlon) * (16 + (lon_stride == 1 ? 2 * (dtype == WB2_F32 ? 4 : 8) : 0));
    tile = lon_stride == 1 ? 1 : eke_tile(nlon, max_smem);
    WB2_REQUIRE(tile > 0 && row_bytes + 16384 <= size_t(max_smem),
                "wb2_column_integral: a row of nlon = %d cells needs %zu B of shared memory",
                nlon, row_bytes);
  }

  Packer pk(ctx);
  const size_t o_w = nlev > 1 ? pk.add(weight, size_t(nlev - 1) * sizeof(double)) : 0;
  WB2_TRY(pk.commit());
  const double* w = nlev > 1 ? pk.dev<double>(o_w) : nullptr;
  int rc;
  if (dtype == WB2_F32)
    rc = launch(ctx, kind, static_cast<const float*>(q), static_cast<const float*>(u),
                static_cast<const float*>(v), nouter, outer_stride, nlev, ninner, nlon, lon_stride,
                tile, w, static_cast<float*>(out));
  else
    rc = launch(ctx, kind, static_cast<const double*>(q), static_cast<const double*>(u),
                static_cast<const double*>(v), nouter, outer_stride, nlev, ninner, nlon,
                lon_stride, tile, w, static_cast<double*>(out));
  if (rc != WB2_OK) return rc;
  return pk.release();
}

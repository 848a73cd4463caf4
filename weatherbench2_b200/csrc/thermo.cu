// Thermodynamic derived variables (sm_90a): the lapse rate and the relative
// humidity of weatherbench2/derived_variables.py:341-362 and 433-468.
//
// Lapse rate  dT_dp / dz_dp with dT_dp = differentiate(T, 'level') and
//   dz_dp = (1 / 9.81) * differentiate(Z, 'level'): np.gradient along the level
//   axis (gradient.cuh), then a multiplication and a division in the data type.
//   One thread per (outer, inner) column walks the column's levels, holding a
//   three-level window of T and Z in registers; consecutive threads take
//   consecutive inner cells, so every load of a warp is coalesced.  When the
//   inner extent is below a warp (the level axis innermost) one thread per
//   cell reads its stencil instead, so a warp's loads stay contiguous.
// Relative humidity  mixing_ratio / saturation_mixing_ratio, elementwise, with
//   the pressure coordinate broadcast along one axis of the layout.  In the
//   slab path a CTA row covers one (outer, p) slab, so the pressure is the same
//   for the whole CTA and no per-element index division is needed; when the
//   pressure axis is (nearly) innermost the slabs are too short for that and
//   each thread finds its pressure by division instead.
// The arithmetic steps follow NumPy's dtypes exactly and use correctly rounded
// intrinsics only (include/wb2b200.h lists them).
#include <algorithm>

#include "common.cuh"
#include "gradient.cuh"

namespace wb2 {
namespace {

constexpr double kInvG = 1 / 9.81;  // `(1 / g)` in derived_variables.py:360
constexpr int kThreads = 256;
constexpr int kIlp = 4;  // elements per thread in flight in the RH kernel

__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float div_rn(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double div_rn(double a, double b) { return __ddiv_rn(a, b); }
using grad::sub_rn;

// exp of the Bolton formula: a float32 argument is evaluated in float64 and
// rounded once; a float64 argument takes CUDA's exp (at most 1 ulp off).
__device__ __forceinline__ float bolton_exp(float x) { return __double2float_rn(exp(double(x))); }
__device__ __forceinline__ double bolton_exp(double x) { return exp(x); }

template <typename T>
__device__ __forceinline__ T load(const T* p) {
  return ldg_stream(p);
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
    lapse_rate_kernel(const T* __restrict__ t, const T* __restrict__ z, int64_t nouter,
                      int32_t nlev, int64_t ninner, const double* __restrict__ coef,
                      int uniform, T* __restrict__ out) {
  const T inv_g = T(kInvG);
  const int64_t cell = int64_t(blockIdx.x) * kThreads + threadIdx.x;
  if (cell < nouter * ninner) {
    const int64_t o = cell / ninner;
    int64_t at = o * nlev * ninner + (cell - o * ninner);
    // window of levels k-1, k, k+1 (tm / zm unused at k = 0)
    T tm = T(0), zm = T(0);
    T t0 = load(t + at), z0 = load(z + at);
    T tp = load(t + at + ninner), zp = load(z + at + ninner);
    for (int k = 0; k < nlev; ++k) {
      const T dt = grad::at_index(tm, t0, tp, k, nlev, coef, uniform != 0);
      const T dz = mul_rn(inv_g, grad::at_index(zm, z0, zp, k, nlev, coef, uniform != 0));
      out[at] = div_rn(dt, dz);
      tm = t0;
      zm = z0;
      t0 = tp;
      z0 = zp;
      at += ninner;
      if (k + 2 < nlev) {
        tp = load(t + at + ninner);
        zp = load(z + at + ninner);
      }
    }
  }
}

// Short columns' inner extent (ninner < 32, e.g. the level axis innermost): a
// warp would read addresses nlev * ninner apart, so instead each thread takes
// one cell and reads the stencil's neighbours, which L1 serves to the adjacent
// threads that also read them.
template <typename T>
__global__ void __launch_bounds__(kThreads)
    lapse_rate_cell_kernel(const T* __restrict__ t, const T* __restrict__ z, int64_t n,
                           int32_t nlev, int64_t ninner, const double* __restrict__ coef,
                           int uniform, T* __restrict__ out) {
  const int64_t i = int64_t(blockIdx.x) * kThreads + threadIdx.x;
  if (i < n) {
    const int k = static_cast<int>((i / ninner) % nlev);
    const T dt = gradient(t + i, k, nlev, ninner, coef, uniform != 0);
    const T dz = mul_rn(T(kInvG), gradient(z + i, k, nlev, ninner, coef, uniform != 0));
    out[i] = div_rn(dt, dz);
  }
}

template <typename T, typename O>
__device__ __forceinline__ O relative_humidity(T t, T q, O p) {
  const T x = div_rn(mul_rn(T(17.67), sub_rn(t, T(273.15))), sub_rn(t, T(29.65)));
  const T svp = mul_rn(T(6.112), bolton_exp(x));
  const T mr = div_rn(q, sub_rn(T(1), q));
  const O smr = div_rn(O(mul_rn(T(0.622), svp)), sub_rn(p, O(svp)));
  return div_rn(O(mr), smr);
}

// Slab path: blockIdx.y walks the (outer, p) slabs of ninner cells, the CTAs of
// one grid row share a slab, and each thread keeps kIlp loads in flight.
template <typename T, typename O>
__global__ void __launch_bounds__(kThreads)
    rh_slab_kernel(const T* __restrict__ t, const T* __restrict__ q, int64_t nslab,
                   int32_t npres, int64_t ninner, const double* __restrict__ pressure,
                   O* __restrict__ out) {
  const int64_t step = int64_t(gridDim.x) * kThreads;
  for (int64_t slab = blockIdx.y; slab < nslab; slab += gridDim.y) {
    const O p = O(__ldg(pressure + slab % npres));
    const int64_t base = slab * ninner;
    for (int64_t i0 = int64_t(blockIdx.x) * kThreads + threadIdx.x; i0 < ninner;
         i0 += kIlp * step) {
      T tv[kIlp], qv[kIlp];
#pragma unroll
      for (int j = 0; j < kIlp; ++j) {
        const int64_t i = i0 + j * step;
        tv[j] = i < ninner ? load(t + base + i) : T(0);
        qv[j] = i < ninner ? load(q + base + i) : T(0);
      }
#pragma unroll
      for (int j = 0; j < kIlp; ++j) {
        const int64_t i = i0 + j * step;
        if (i < ninner) out[base + i] = relative_humidity(tv[j], qv[j], p);
      }
    }
  }
}

// Short slabs (the pressure axis innermost or nearly so): a flat grid-stride
// loop, the pressure index found per element.
template <typename T, typename O>
__global__ void __launch_bounds__(kThreads)
    rh_flat_kernel(const T* __restrict__ t, const T* __restrict__ q, int64_t n,
                   int32_t npres, int64_t ninner, const double* __restrict__ pressure,
                   O* __restrict__ out) {
  for (int64_t i = int64_t(blockIdx.x) * kThreads + threadIdx.x; i < n;
       i += int64_t(gridDim.x) * kThreads) {
    const O p = O(__ldg(pressure + (i / ninner) % npres));
    out[i] = relative_humidity(load(t + i), load(q + i), p);
  }
}

template <typename T>
int launch_lapse(wb2_ctx* ctx, const void* t, const void* z, int64_t nouter, int32_t nlev,
                 int64_t ninner, const double* coef, int uniform, void* out) {
  const T* tp = static_cast<const T*>(t);
  const T* zp = static_cast<const T*>(z);
  T* op = static_cast<T*>(out);
  if (ninner < 32) {  // one thread per cell
    const int64_t n = nouter * nlev * ninner;
    const int64_t nblk = (n + kThreads - 1) / kThreads;
    WB2_REQUIRE(nblk <= INT32_MAX, "wb2_lapse_rate: too many cells for the grid");
    return launch_kernel(ctx, lapse_rate_cell_kernel<T>, dim3(static_cast<unsigned>(nblk)),
                         kThreads, 0, tp, zp, n, nlev, ninner, coef, uniform, op);
  }
  const int64_t nblk = (nouter * ninner + kThreads - 1) / kThreads;  // one thread per column
  WB2_REQUIRE(nblk <= INT32_MAX, "wb2_lapse_rate: too many columns for the grid");
  return launch_kernel(ctx, lapse_rate_kernel<T>, dim3(static_cast<unsigned>(nblk)), kThreads,
                       0, tp, zp, nouter, nlev, ninner, coef, uniform, op);
}

template <typename T, typename O>
int launch_rh(wb2_ctx* ctx, const void* t, const void* q, int64_t nouter, int32_t npres,
              int64_t ninner, const double* pressure, void* out) {
  const int64_t nslab = nouter * npres;
  const int64_t want = int64_t(ctx->num_sms) * 16;  // CTAs: 16 per SM, in flight
  const T* tp = static_cast<const T*>(t);
  const T* qp = static_cast<const T*>(q);
  O* op = static_cast<O*>(out);
  if (ninner >= kThreads) {
    const int64_t gy = std::min<int64_t>(nslab, 65535);
    const int64_t gx = std::max<int64_t>(
        1, std::min<int64_t>((ninner + kThreads - 1) / kThreads, (want + gy - 1) / gy));
    return launch_kernel(ctx, rh_slab_kernel<T, O>,
                         dim3(static_cast<unsigned>(gx), static_cast<unsigned>(gy)), kThreads,
                         0, tp, qp, nslab, npres, ninner, pressure, op);
  }
  const int64_t n = nslab * ninner;
  const int64_t nblk = std::min<int64_t>((n + kThreads - 1) / kThreads, want);
  return launch_kernel(ctx, rh_flat_kernel<T, O>, dim3(static_cast<unsigned>(nblk)), kThreads,
                       0, tp, qp, n, npres, ninner, pressure, op);
}

}  // namespace
}  // namespace wb2

using namespace wb2;

extern "C" int wb2_lapse_rate(wb2_ctx* ctx, int dtype, const void* t, const void* z,
                              int64_t nouter, int32_t nlev, int64_t ninner, const double* coef,
                              int uniform, void* out) {
  WB2_NVTX("wb2_lapse_rate");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_REQUIRE(dtype == WB2_F32 || dtype == WB2_F64, "wb2_lapse_rate: unknown dtype %d", dtype);
  WB2_REQUIRE(nouter >= 0 && nlev >= 0 && ninner >= 0, "wb2_lapse_rate: negative size");
  WB2_REQUIRE(nlev >= 2,
              "wb2_lapse_rate: need at least 2 levels to take a gradient (nlev=%d)", nlev);
  WB2_REQUIRE(t != nullptr && z != nullptr && out != nullptr && coef != nullptr,
              "wb2_lapse_rate: NULL argument");
  if (nouter == 0 || ninner == 0) return WB2_OK;
  DeviceGuard guard(ctx->device);
  Packer pk(ctx);
  const size_t o_c = pk.add(coef, size_t(nlev) * 3 * sizeof(double));
  WB2_TRY(pk.commit());
  const double* c = pk.dev<double>(o_c);
  WB2_TRY(dtype == WB2_F32 ? launch_lapse<float>(ctx, t, z, nouter, nlev, ninner, c, uniform, out)
                           : launch_lapse<double>(ctx, t, z, nouter, nlev, ninner, c, uniform, out));
  ctx->launches += 1;
  return pk.release();
}

extern "C" int wb2_relative_humidity(wb2_ctx* ctx, int dtype, int out_dtype, const void* t,
                                     const void* q, int64_t nouter, int32_t npres,
                                     int64_t ninner, const double* pressure, void* out) {
  WB2_NVTX("wb2_relative_humidity");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_REQUIRE(dtype == WB2_F32 || dtype == WB2_F64, "wb2_relative_humidity: unknown dtype %d",
              dtype);
  WB2_REQUIRE(out_dtype == WB2_F32 || out_dtype == WB2_F64,
              "wb2_relative_humidity: unknown out_dtype %d", out_dtype);
  WB2_REQUIRE(!(dtype == WB2_F64 && out_dtype == WB2_F32),
              "wb2_relative_humidity: out_dtype float32 is narrower than float64 data");
  WB2_REQUIRE(nouter >= 0 && npres >= 1 && ninner >= 0,
              "wb2_relative_humidity: negative size or npres < 1");
  WB2_REQUIRE(t != nullptr && q != nullptr && out != nullptr && pressure != nullptr,
              "wb2_relative_humidity: NULL argument");
  if (nouter == 0 || ninner == 0) return WB2_OK;
  DeviceGuard guard(ctx->device);
  Packer pk(ctx);
  const size_t o_p = pk.add(pressure, size_t(npres) * sizeof(double));
  WB2_TRY(pk.commit());
  const double* p = pk.dev<double>(o_p);
  int rc;
  if (dtype == WB2_F64)
    rc = launch_rh<double, double>(ctx, t, q, nouter, npres, ninner, p, out);
  else if (out_dtype == WB2_F64)
    rc = launch_rh<float, double>(ctx, t, q, nouter, npres, ninner, p, out);
  else
    rc = launch_rh<float, float>(ctx, t, q, nouter, npres, ninner, p, out);
  WB2_TRY(rc);
  ctx->launches += 1;
  return pk.release();
}

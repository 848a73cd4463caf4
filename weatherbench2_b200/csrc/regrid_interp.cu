// K8 -- nearest-neighbour and bilinear regridding (sm_90a).
//
// wb2_regrid_gather replaces NearestRegridder.regrid_array
// (weatherbench2/regridding.py:231-247): out[k] = src.ravel()[indices[k]] with the
// BallTree / haversine indices computed once on the host exactly like the
// reference (:212-228).
//
// wb2_regrid_bilinear replaces BilinearRegridder.regrid_array (:256-294): two
// 1-D linear interpolations with jnp.interp's formula
//     f = fp[i-1] + (delta / dx) * (fp[i] - fp[i-1])
// first along latitude, then along longitude, in float32 like JAX.  The host
// resolves x % period / the stable key sort / searchsorted / the clip into two
// taps and the fraction t = delta / dx per target coordinate (i0 = -1: NaN, the
// left = right = nan `where`s).  jnp.interp's other `where`s -- fp[0] / fp[-1]
// outside a clamped axis, fp[i-1] where |dx| <= spacing(eps) -- return the tap
// value itself; the host marks them i1 = i0, t = -1 and the kernel passes
// fp[i0] through untouched, so an infinite tap stays infinite (fp + 0 * (fp - fp)
// would be NaN).  A genuine fraction is never negative (it lies in [0, 1], -0.0
// at most), and i1 = i0 with t = -1 read as a plain lerp still gives
// fp + (-1) * 0 = fp bit for bit for every finite tap, -0.0 included.
// Each lerp is three separately rounded operations (no FMA contraction), so
// given the host's taps the result is bit-equal to a float32 transcription of
// jnp.interp applied in the reference's order.
//
// Fields are (lon, lat) slabs like the conservative regridder's.  Both kernels
// are gathers: 4 B written per target cell, 4 (nearest) or 16 (bilinear) bytes
// read per target cell from rows that stay in L2.
#include <algorithm>

#include "common.cuh"

namespace wb2 {

constexpr int kInterpThreads = 256;

// jnp.interp's a + t * (b - a), each operation rounded on its own
__device__ __forceinline__ float lerp_rn(float a, float b, float t) {
  return __fadd_rn(a, __fmul_rn(t, __fsub_rn(b, a)));
}

__global__ void __launch_bounds__(kInterpThreads)
    regrid_gather_kernel(const float* __restrict__ src, float* __restrict__ dst,
                         const int32_t* __restrict__ idx, int64_t src_stride, int64_t dst_stride,
                         int32_t ntarget) {
  const int64_t field = blockIdx.y;
  const int k = blockIdx.x * kInterpThreads + threadIdx.x;
  if (k >= ntarget) return;
  dst[field * dst_stride + k] = __ldg(src + field * src_stride + idx[k]);
}

struct BilinearParams {
  const float* src;
  float* dst;
  const int32_t* lon_i0;  // [nlon_t] source longitude index of the left tap, -1: NaN
  const int32_t* lon_i1;  // right tap (-1 exactly where lon_i0 is)
  const float* lon_t;     // [nlon_t] delta / dx; < 0: fp[lon_i0] exactly
  const int32_t* lat_i0;  // [nlat_t]
  const int32_t* lat_i1;
  const float* lat_t;
  int64_t src_stride, dst_stride;
  int32_t nlon_t, nlat_t, nlat_s;
};

__global__ void __launch_bounds__(kInterpThreads) regrid_bilinear_kernel(const BilinearParams p) {
  const int64_t field = blockIdx.y;
  const int k = blockIdx.x * kInterpThreads + threadIdx.x;
  if (k >= p.nlon_t * p.nlat_t) return;
  const int a = k / p.nlat_t;  // target longitude
  const int c = k - a * p.nlat_t;
  const int b0 = p.lon_i0[a], b1 = p.lon_i1[a];
  const int d0 = p.lat_i0[c], d1 = p.lat_i1[c];
  float out = __int_as_float(0x7fc00000);
  if (b0 >= 0 && d0 >= 0) {
    const float* s = p.src + field * p.src_stride;
    const float tl = p.lat_t[c], tn = p.lon_t[a];
    // latitude first (regridding.py:262-274), on the two longitude taps; a
    // negative fraction returns the i0 tap itself (jnp.interp's `where`)
    const float x00 = __ldg(s + int64_t(b0) * p.nlat_s + d0);
    const float x01 = __ldg(s + int64_t(b0) * p.nlat_s + d1);
    const float x10 = __ldg(s + int64_t(b1) * p.nlat_s + d0);
    const float x11 = __ldg(s + int64_t(b1) * p.nlat_s + d1);
    const float y0 = tl < 0.f ? x00 : lerp_rn(x00, x01, tl);
    const float y1 = tl < 0.f ? x10 : lerp_rn(x10, x11, tl);
    out = tn < 0.f ? y0 : lerp_rn(y0, y1, tn);  // then longitude (:276-292)
  }
  p.dst[field * p.dst_stride + k] = out;
}

}  // namespace wb2

using namespace wb2;

extern "C" int wb2_regrid_gather(wb2_ctx* ctx, const float* src, float* dst, int64_t nfield,
                                 int64_t src_field_stride, int64_t dst_field_stride,
                                 int32_t nsource, int32_t ntarget, const int32_t* indices) {
  WB2_NVTX("wb2_regrid_gather");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_REQUIRE(nfield >= 0 && nfield < 65536LL * 65536LL, "nfield out of range");
  WB2_REQUIRE(nsource > 0 && ntarget > 0, "empty grid");
  if (nfield == 0) return WB2_OK;
  WB2_REQUIRE(src && dst && indices, "NULL argument");
  for (int32_t k = 0; k < ntarget; ++k)
    WB2_REQUIRE(indices[k] >= 0 && indices[k] < nsource, "indices[%d] = %d out of range", k,
                indices[k]);
  DeviceGuard guard(ctx->device);
  Packer pk(ctx);
  const size_t o = pk.add(indices, size_t(ntarget) * sizeof(int32_t));
  WB2_TRY(pk.commit());
  const unsigned bx = (ntarget + kInterpThreads - 1) / kInterpThreads;
  for (int64_t f0 = 0; f0 < nfield; f0 += 65535) {
    const unsigned by = static_cast<unsigned>(std::min<int64_t>(65535, nfield - f0));
    regrid_gather_kernel<<<dim3(bx, by), kInterpThreads, 0, ctx->stream>>>(
        src + f0 * src_field_stride, dst + f0 * dst_field_stride, pk.dev<int32_t>(o),
        src_field_stride, dst_field_stride, ntarget);
    WB2_CUDA_TRY(cudaGetLastError());
    ctx->launches += 1;
  }
  WB2_TRY(pk.release());
  return WB2_OK;
}

extern "C" int wb2_regrid_bilinear(wb2_ctx* ctx, const float* src, float* dst, int64_t nfield,
                                   int64_t src_field_stride, int64_t dst_field_stride,
                                   int32_t nlon_s, int32_t nlat_s, int32_t nlon_t, int32_t nlat_t,
                                   const int32_t* lon_i0, const int32_t* lon_i1,
                                   const float* lon_t, const int32_t* lat_i0,
                                   const int32_t* lat_i1, const float* lat_t) {
  WB2_NVTX("wb2_regrid_bilinear");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_REQUIRE(nfield >= 0 && nfield < 65536LL * 65536LL, "nfield out of range");
  WB2_REQUIRE(nlon_s > 0 && nlat_s > 0 && nlon_t > 0 && nlat_t > 0, "empty grid");
  if (nfield == 0) return WB2_OK;
  WB2_REQUIRE(src && dst && lon_i0 && lon_i1 && lon_t && lat_i0 && lat_i1 && lat_t,
              "NULL argument");
  for (int32_t a = 0; a < nlon_t; ++a)
    WB2_REQUIRE(lon_i0[a] >= -1 && lon_i0[a] < nlon_s && lon_i1[a] >= -1 && lon_i1[a] < nlon_s &&
                    (lon_i0[a] < 0) == (lon_i1[a] < 0),
                "longitude tap %d out of range", a);
  for (int32_t c = 0; c < nlat_t; ++c)
    WB2_REQUIRE(lat_i0[c] >= -1 && lat_i0[c] < nlat_s && lat_i1[c] >= -1 && lat_i1[c] < nlat_s &&
                    (lat_i0[c] < 0) == (lat_i1[c] < 0),
                "latitude tap %d out of range", c);
  DeviceGuard guard(ctx->device);
  Packer pk(ctx);
  const size_t o0 = pk.add(lon_i0, size_t(nlon_t) * sizeof(int32_t));
  const size_t o1 = pk.add(lon_i1, size_t(nlon_t) * sizeof(int32_t));
  const size_t o2 = pk.add(lon_t, size_t(nlon_t) * sizeof(float));
  const size_t o3 = pk.add(lat_i0, size_t(nlat_t) * sizeof(int32_t));
  const size_t o4 = pk.add(lat_i1, size_t(nlat_t) * sizeof(int32_t));
  const size_t o5 = pk.add(lat_t, size_t(nlat_t) * sizeof(float));
  WB2_TRY(pk.commit());
  BilinearParams p;
  p.lon_i0 = pk.dev<int32_t>(o0); p.lon_i1 = pk.dev<int32_t>(o1); p.lon_t = pk.dev<float>(o2);
  p.lat_i0 = pk.dev<int32_t>(o3); p.lat_i1 = pk.dev<int32_t>(o4); p.lat_t = pk.dev<float>(o5);
  p.src_stride = src_field_stride; p.dst_stride = dst_field_stride;
  p.nlon_t = nlon_t; p.nlat_t = nlat_t; p.nlat_s = nlat_s;
  const unsigned bx = (nlon_t * nlat_t + kInterpThreads - 1) / kInterpThreads;
  for (int64_t f0 = 0; f0 < nfield; f0 += 65535) {
    const unsigned by = static_cast<unsigned>(std::min<int64_t>(65535, nfield - f0));
    p.src = src + f0 * src_field_stride;
    p.dst = dst + f0 * dst_field_stride;
    regrid_bilinear_kernel<<<dim3(bx, by), kInterpThreads, 0, ctx->stream>>>(p);
    WB2_CUDA_TRY(cudaGetLastError());
    ctx->launches += 1;
  }
  WB2_TRY(pk.release());
  return WB2_OK;
}

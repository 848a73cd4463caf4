// Horizontal-derivative diagnostics of the wind and geopotential (sm_90a):
// divergence, vorticity, vertical velocity and the geostrophic / ageostrophic
// winds of weatherbench2/derived_variables.py:102-338, one kernel per `kind`.
//
// The reference builds all nine on xarray's `differentiate`, i.e.
// np.gradient(f, coord, edge_order=1), and the two operators
//   _d_dx(f) = where(cos(lat) > 1e-6, g_lon(f) / cos(lat) / M, 0)   (float64)
//   _d_dy(f) = g_lat(f) / M                                          (float32)
// with M = 2 pi 6367500 / 360 metres per degree.  Every step below is the
// operation NumPy performs on float32 data and float64 coordinates, correctly
// rounded and never contracted into an FMA, so each output is the reference's
// float64 result rounded once to float32:
//   g (np.gradient, stored as float32): edges (f[1] - f[0]) / dx[0] and
//     (f[n-1] - f[n-2]) / dx[n-2]; uniform interior (f[i+1] - f[i-1]) / (2 dx);
//     otherwise a f[i-1] + b f[i] + c f[i+1] in float64, left to right.  The
//     float32 differences are float32 subtractions, the divisions float64.
//   geostrophic u = -_d_dy(z) / f, v = _d_dx(z) / f (f = 2 Omega sin(lat); inf /
//   NaN on the equator, as in the reference), speeds sqrt(u*u + v*v), the
//   ageostrophic wind u - u_geo, all in float64.
//   vertical velocity: scipy's cumulative_trapezoid(-div, x=100*level,
//   initial=0) -- cumsum(dp_k * (y[k+1] + y[k]) / 2.0) -- walked by one thread
//   per column over the float64 divergence, which is never rounded.
// The host supplies the per-index gradient coefficients, cos(lat), f and the
// pressures, computed by the same NumPy expressions as the reference.
//
// Threads map to consecutive addresses of a field in either layout ((lat, lon)
// or (lon, lat)); the neighbour rows a stencil reads come back from L1 / L2
// (DESIGN.md, "Wind dynamics", has the measurement).
#include <algorithm>

#include "common.cuh"
#include "gradient.cuh"

namespace wb2 {
namespace {

constexpr double kMetersPerDegree = 2 * 3.141592653589793 * 6367500.0 / 360;  // schema.py:59
constexpr float kMetersPerDegreeF = static_cast<float>(kMetersPerDegree);
constexpr int kThreads = 256;

struct DynParams {
  const float* u;
  const float* v;
  const float* z;
  float* out;
  int64_t nfield;    // fields of nlat * nlon cells (columns of nlev fields for kind 2)
  int32_t nlev;
  int32_t nlat, nlon;
  int32_t lon_contig;  // 1: (lat, lon) layout; 0: (lon, lat)
  int32_t lat_uniform, lon_uniform;
  const double* lat_coef;  // [nlat][3]
  const double* lon_coef;  // [nlon][3]
  const double* cos_lat;   // [nlat]
  const double* coriolis;  // [nlat]
  const double* pressure;  // [nlev]
};

// np.gradient(f, x, edge_order=1) is gradient<float>() of gradient.cuh: each
// derivative rounded to float32 as np.gradient stores it.

// the reference's _d_dx (float64) and _d_dy (float32)
__device__ __forceinline__ double d_dx(float g, double cos_lat) {
  return cos_lat > 1e-6 ? __ddiv_rn(__ddiv_rn(double(g), cos_lat), kMetersPerDegree) : 0.0;
}
__device__ __forceinline__ float d_dy(float g) { return __fdiv_rn(g, kMetersPerDegreeF); }

__device__ __forceinline__ double hypot_rn(double a, double b) {
  return __dsqrt_rn(__dadd_rn(__dmul_rn(a, a), __dmul_rn(b, b)));
}

struct Cell {
  int ilat, ilon;
  int64_t lat_s, lon_s;
};

__device__ __forceinline__ float g_lon(const DynParams& p, const float* f, const Cell& c) {
  return gradient(f, c.ilon, p.nlon, c.lon_s, p.lon_coef, p.lon_uniform);
}
__device__ __forceinline__ float g_lat(const DynParams& p, const float* f, const Cell& c) {
  return gradient(f, c.ilat, p.nlat, c.lat_s, p.lat_coef, p.lat_uniform);
}

// divergence _d_dx(u) + _d_dy(v), float64
__device__ __forceinline__ double divergence(const DynParams& p, int64_t at, const Cell& c,
                                             double cosv) {
  return __dadd_rn(d_dx(g_lon(p, p.u + at, c), cosv), double(d_dy(g_lat(p, p.v + at, c))));
}

template <int KIND>
__global__ void __launch_bounds__(kThreads) wind_dynamics_kernel(const DynParams p) {
  const int32_t ncell = p.nlat * p.nlon;
  const int32_t t = blockIdx.x * kThreads + threadIdx.x;
  if (t >= ncell) return;
  Cell c;
  if (p.lon_contig) {
    c.ilat = t / p.nlon;
    c.ilon = t - c.ilat * p.nlon;
    c.lat_s = p.nlon;
    c.lon_s = 1;
  } else {
    c.ilon = t / p.nlat;
    c.ilat = t - c.ilon * p.nlat;
    c.lat_s = 1;
    c.lon_s = p.nlat;
  }
  const double cosv = __ldg(p.cos_lat + c.ilat);
  for (int64_t field = blockIdx.y; field < p.nfield; field += gridDim.y) {
    if constexpr (KIND == WB2_DYN_VERTICAL_VELOCITY) {
      // one column: levels k = 0 .. nlev-1 of outer index `field`
      const int64_t step = int64_t(ncell);
      int64_t at = field * p.nlev * step + t;
      double prev = divergence(p, at, c, cosv);
      double pprev = __ldg(p.pressure);
      double acc = 0.0;
      p.out[at] = 0.0f;
      for (int k = 1; k < p.nlev; ++k) {
        at += step;
        const double cur = divergence(p, at, c, cosv);
        const double pk = __ldg(p.pressure + k);
        // cumulative_trapezoid of y = -div: d * (y[k] + y[k-1]) / 2.0
        const double term =
            __ddiv_rn(__dmul_rn(__dsub_rn(pk, pprev), __dadd_rn(-cur, -prev)), 2.0);
        acc = k == 1 ? term : __dadd_rn(acc, term);
        p.out[at] = __double2float_rn(acc);
        prev = cur;
        pprev = pk;
      }
    } else {
      const int64_t at = field * int64_t(ncell) + t;
      double r;
      if constexpr (KIND == WB2_DYN_DIVERGENCE) {
        r = divergence(p, at, c, cosv);
      } else if constexpr (KIND == WB2_DYN_VORTICITY) {
        r = __dsub_rn(d_dx(g_lon(p, p.v + at, c), cosv), double(d_dy(g_lat(p, p.u + at, c))));
      } else {
        const double f = __ldg(p.coriolis + c.ilat);
        constexpr bool need_u = KIND != WB2_DYN_V_GEOSTROPHIC && KIND != WB2_DYN_V_AGEOSTROPHIC;
        constexpr bool need_v = KIND != WB2_DYN_U_GEOSTROPHIC && KIND != WB2_DYN_U_AGEOSTROPHIC;
        double ug = 0.0, vg = 0.0;
        if constexpr (need_u) ug = __ddiv_rn(double(-d_dy(g_lat(p, p.z + at, c))), f);
        if constexpr (need_v) vg = __ddiv_rn(d_dx(g_lon(p, p.z + at, c), cosv), f);
        if constexpr (KIND == WB2_DYN_GEOSTROPHIC_WIND_SPEED) r = hypot_rn(ug, vg);
        if constexpr (KIND == WB2_DYN_U_GEOSTROPHIC) r = ug;
        if constexpr (KIND == WB2_DYN_V_GEOSTROPHIC) r = vg;
        if constexpr (KIND == WB2_DYN_AGEOSTROPHIC_WIND_SPEED)
          r = hypot_rn(__dsub_rn(double(__ldg(p.u + at)), ug),
                       __dsub_rn(double(__ldg(p.v + at)), vg));
        if constexpr (KIND == WB2_DYN_U_AGEOSTROPHIC) r = __dsub_rn(double(__ldg(p.u + at)), ug);
        if constexpr (KIND == WB2_DYN_V_AGEOSTROPHIC) r = __dsub_rn(double(__ldg(p.v + at)), vg);
      }
      p.out[at] = __double2float_rn(r);
    }
  }
}

template <int KIND>
int launch(wb2_ctx* ctx, const DynParams& p) {
  const int32_t ncell = p.nlat * p.nlon;
  const unsigned gx = static_cast<unsigned>((ncell + kThreads - 1) / kThreads);
  // enough CTAs to fill the SMs several times over; more fields loop in-kernel
  const int64_t want = std::max<int64_t>(1, int64_t(ctx->num_sms) * 32 / gx);
  const unsigned gy = static_cast<unsigned>(std::min<int64_t>({p.nfield, want, 65535}));
  wind_dynamics_kernel<KIND><<<dim3(gx, gy), kThreads, 0, ctx->stream>>>(p);
  WB2_CUDA_TRY(cudaGetLastError());
  return WB2_OK;
}

}  // namespace
}  // namespace wb2

using namespace wb2;

extern "C" int wb2_wind_dynamics(wb2_ctx* ctx, int kind, const float* u, const float* v,
                                 const float* z, int64_t nouter, int32_t nlev, int32_t nlat,
                                 int32_t nlon, int64_t lat_stride, int64_t lon_stride,
                                 const double* lat_coef, int lat_uniform, const double* lon_coef,
                                 int lon_uniform, const double* cos_lat, const double* coriolis,
                                 const double* pressure, float* out) {
  WB2_NVTX("wb2_wind_dynamics");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_REQUIRE(kind >= WB2_DYN_DIVERGENCE && kind <= WB2_DYN_V_AGEOSTROPHIC,
              "wb2_wind_dynamics: unknown kind %d", kind);
  WB2_REQUIRE(nouter >= 0 && nlev >= 0, "wb2_wind_dynamics: negative size");
  WB2_REQUIRE(nlat >= 2 && nlon >= 2,
              "wb2_wind_dynamics: need at least 2 points along latitude and longitude "
              "(nlat=%d, nlon=%d)", nlat, nlon);
  WB2_REQUIRE(int64_t(nlat) * nlon <= INT32_MAX, "wb2_wind_dynamics: field too large");
  const bool lon_contig = lon_stride == 1 && lat_stride == nlon;
  WB2_REQUIRE(lon_contig || (lat_stride == 1 && lon_stride == nlat),
              "wb2_wind_dynamics: strides (lat %lld, lon %lld) are neither (nlon, 1) nor (1, nlat)",
              static_cast<long long>(lat_stride), static_cast<long long>(lon_stride));
  const bool uses_wind = kind <= WB2_DYN_VERTICAL_VELOCITY || kind >= WB2_DYN_AGEOSTROPHIC_WIND_SPEED;
  const bool uses_z = kind >= WB2_DYN_GEOSTROPHIC_WIND_SPEED;
  WB2_REQUIRE(out && lat_coef && lon_coef && cos_lat, "wb2_wind_dynamics: NULL argument");
  WB2_REQUIRE(!uses_z || (z && coriolis), "wb2_wind_dynamics: NULL z or coriolis");
  WB2_REQUIRE(!uses_wind || kind == WB2_DYN_V_AGEOSTROPHIC || u, "wb2_wind_dynamics: NULL u");
  WB2_REQUIRE(!uses_wind || kind == WB2_DYN_U_AGEOSTROPHIC || v, "wb2_wind_dynamics: NULL v");
  WB2_REQUIRE(kind != WB2_DYN_VERTICAL_VELOCITY || pressure,
              "wb2_wind_dynamics: NULL pressure");
  if (nouter == 0 || nlev == 0) return WB2_OK;
  DeviceGuard guard(ctx->device);

  Packer pk(ctx);
  const size_t o_lat = pk.add(lat_coef, size_t(nlat) * 3 * sizeof(double));
  const size_t o_lon = pk.add(lon_coef, size_t(nlon) * 3 * sizeof(double));
  const size_t o_cos = pk.add(cos_lat, size_t(nlat) * sizeof(double));
  const size_t o_cor = uses_z ? pk.add(coriolis, size_t(nlat) * sizeof(double)) : 0;
  const size_t o_p =
      kind == WB2_DYN_VERTICAL_VELOCITY ? pk.add(pressure, size_t(nlev) * sizeof(double)) : 0;
  WB2_TRY(pk.commit());
  DynParams p;
  p.u = u;
  p.v = v;
  p.z = z;
  p.out = out;
  p.nfield = kind == WB2_DYN_VERTICAL_VELOCITY ? nouter : nouter * nlev;
  p.nlev = nlev;
  p.nlat = nlat;
  p.nlon = nlon;
  p.lon_contig = lon_contig;
  p.lat_uniform = lat_uniform != 0;
  p.lon_uniform = lon_uniform != 0;
  p.lat_coef = pk.dev<double>(o_lat);
  p.lon_coef = pk.dev<double>(o_lon);
  p.cos_lat = pk.dev<double>(o_cos);
  p.coriolis = uses_z ? pk.dev<double>(o_cor) : nullptr;
  p.pressure = kind == WB2_DYN_VERTICAL_VELOCITY ? pk.dev<double>(o_p) : nullptr;
  int rc = WB2_OK;
  switch (kind) {
    case WB2_DYN_DIVERGENCE: rc = launch<WB2_DYN_DIVERGENCE>(ctx, p); break;
    case WB2_DYN_VORTICITY: rc = launch<WB2_DYN_VORTICITY>(ctx, p); break;
    case WB2_DYN_VERTICAL_VELOCITY: rc = launch<WB2_DYN_VERTICAL_VELOCITY>(ctx, p); break;
    case WB2_DYN_GEOSTROPHIC_WIND_SPEED: rc = launch<WB2_DYN_GEOSTROPHIC_WIND_SPEED>(ctx, p); break;
    case WB2_DYN_U_GEOSTROPHIC: rc = launch<WB2_DYN_U_GEOSTROPHIC>(ctx, p); break;
    case WB2_DYN_V_GEOSTROPHIC: rc = launch<WB2_DYN_V_GEOSTROPHIC>(ctx, p); break;
    case WB2_DYN_AGEOSTROPHIC_WIND_SPEED: rc = launch<WB2_DYN_AGEOSTROPHIC_WIND_SPEED>(ctx, p); break;
    case WB2_DYN_U_AGEOSTROPHIC: rc = launch<WB2_DYN_U_AGEOSTROPHIC>(ctx, p); break;
    default: rc = launch<WB2_DYN_V_AGEOSTROPHIC>(ctx, p); break;
  }
  if (rc != WB2_OK) return rc;
  ctx->launches += 1;
  return pk.release();
}

// Device-side preprocessing that feeds the metric kernels without a host
// round trip (SURVEY.md section 8 f3).
//
// wb2_ens_mean replaces the ensemble-mean pipeline of
// scripts/compute_ensemble_mean.py:110-141 (xbeam.Mean(realization, skipna)):
// out = mean_m x_m per cell (NaN-skipping when skipna), float32 like xarray's
// mean of float32 data.  4 M bytes read + 4 written per cell: a streaming
// kernel, 8 member loads in flight per thread, 128-bit where aligned.
//
// wb2_spectrum_interp replaces interpolate_spectral_frequencies
// (weatherbench2/derived_variables.py:629-682): every latitude row of a zonal
// spectrum lives on its own frequency axis f_k = k / (L * spacing(lat)) (passed
// as a table, the reference's own coordinate values); the rows are
// interpolated linearly to common frequencies, NaN outside the row's range
// (xarray .interp -> scipy interp1d(bounds_error=False)).  The interval and the
// formula are scipy's linear interp1d (_call_linear): lo = clip(searchsorted(x,
// f, side='left'), 1, nk - 1) - 1, so a node x[k] > x[0] is reached from the
// interval below it, and
//     y = ((f - x_lo) / dx) * y_hi + ((x_hi - f) / dx) * y_lo,   dx = x_hi - x_lo
// in float64 with every operation rounded on its own (no FMA contraction).  The
// float64 value is therefore scipy's bit for bit and the float32 result its
// rounding; NaN / inf propagate exactly as in scipy (0 * inf = NaN included).
#include <algorithm>

#include "common.cuh"

namespace wb2 {

template <int VEC, bool SKIPNA>
__global__ void __launch_bounds__(256) ens_mean_kernel(const float* __restrict__ x,
                                                       const int64_t* __restrict__ off,
                                                       float* __restrict__ out, int nmember,
                                                       int64_t member_stride, int64_t slab,
                                                       int64_t nvec_per_field) {
  const int64_t field = blockIdx.y;
  const float* src = x + off[field];
  float* dst = out + field * slab;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec_per_field;
       i += stride) {
    float s[VEC], c[VEC];
#pragma unroll
    for (int k = 0; k < VEC; ++k) s[k] = c[k] = 0.f;
    int m = 0;
    for (; m + 8 <= nmember; m += 8) {
      float v[8][VEC];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float* p = src + int64_t(m + j) * member_stride + i * VEC;
        if (VEC == 4) {
          const float4 q = ldg_stream(reinterpret_cast<const float4*>(p));
          v[j][0] = q.x; v[j][1 % VEC] = q.y; v[j][2 % VEC] = q.z; v[j][3 % VEC] = q.w;
        } else {
          v[j][0] = ldg_stream(p);
        }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int k = 0; k < VEC; ++k) {
          if (SKIPNA) {
            if (v[j][k] == v[j][k]) { s[k] += v[j][k]; c[k] += 1.f; }
          } else {
            s[k] += v[j][k];
          }
        }
    }
    for (; m < nmember; ++m) {
      const float* p = src + int64_t(m) * member_stride + i * VEC;
#pragma unroll
      for (int k = 0; k < VEC; ++k) {
        const float v = ldg_stream(p + k);
        if (SKIPNA) {
          if (v == v) { s[k] += v; c[k] += 1.f; }
        } else {
          s[k] += v;
        }
      }
    }
    const float fm = float(nmember);
#pragma unroll
    for (int k = 0; k < VEC; ++k) dst[i * VEC + k] = SKIPNA ? s[k] / c[k] : s[k] / fm;  // 0/0 = NaN
  }
}

__global__ void __launch_bounds__(256) spectrum_interp_kernel(
    const float* __restrict__ spec, const double* __restrict__ freq_tab,
    const double* __restrict__ freqs, float* __restrict__ out, int64_t nfield, int nrow, int nk,
    int nf) {
  const int64_t total = nfield * nrow * int64_t(nf);
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int j = static_cast<int>(i % nf);
    const int64_t fr = i / nf;  // field * nrow + row
    const int row = static_cast<int>(fr % nrow);
    const double* x = freq_tab + int64_t(row) * nk;  // this latitude's frequency axis
    const double f = freqs[j];
    float r = __int_as_float(0x7fc00000);
    if (f >= x[0] && f <= x[nk - 1]) {
      // the axis is uniform in k: guess the interval, then settle on the table
      // values themselves (the coordinates are the reference's, not k * step)
      // to the largest lo with x[lo] < f (0 when f == x[0])
      const double step = x[1] - x[0];
      int lo = step > 0.0 ? static_cast<int>(floor((f - x[0]) / step)) : 0;
      lo = max(0, min(lo, nk - 2));
      while (lo < nk - 2 && x[lo + 1] < f) ++lo;
      while (lo > 0 && x[lo] >= f) --lo;
      const double x_lo = x[lo], x_hi = x[lo + 1];
      const double y_lo = double(spec[fr * nk + lo]), y_hi = double(spec[fr * nk + lo + 1]);
      const double dx = __dsub_rn(x_hi, x_lo);
      const double w_hi = __ddiv_rn(__dsub_rn(f, x_lo), dx);
      const double w_lo = __ddiv_rn(__dsub_rn(x_hi, f), dx);
      r = __double2float_rn(__dadd_rn(__dmul_rn(w_hi, y_hi), __dmul_rn(w_lo, y_lo)));
    }
    out[i] = r;
  }
}

}  // namespace wb2

using namespace wb2;

extern "C" int wb2_ens_mean(wb2_ctx* ctx, const float* x, int32_t nmember,
                            int64_t member_stride, int64_t nfield, const int64_t* off_x,
                            int64_t slab, int skipna, float* out) {
  WB2_NVTX("wb2_ens_mean");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_REQUIRE(nmember >= 1 && slab >= 0 && nfield >= 0, "bad sizes");
  if (nfield == 0 || slab == 0) return WB2_OK;
  WB2_REQUIRE(x && out && off_x, "NULL argument");
  WB2_REQUIRE(nfield <= 65535, "at most 65535 fields per call (got %lld)",
              static_cast<long long>(nfield));
  DeviceGuard guard(ctx->device);
  bool vec = (slab % 4 == 0) && (member_stride % 4 == 0) &&
             (reinterpret_cast<uintptr_t>(x) & 15) == 0 &&
             (reinterpret_cast<uintptr_t>(out) & 15) == 0;
  for (int64_t i = 0; vec && i < nfield; ++i) vec = off_x[i] % 4 == 0;
  Packer pk(ctx);
  const size_t o = pk.add(off_x, size_t(nfield) * sizeof(int64_t));
  WB2_TRY(pk.commit());
  const int64_t nvec = vec ? slab / 4 : slab;
  const unsigned bx = static_cast<unsigned>(
      std::max<int64_t>(1, std::min<int64_t>((nvec + 255) / 256,
                                             std::max<int64_t>(1, int64_t(ctx->num_sms) * 8 / nfield))));
  const dim3 grid(bx, static_cast<unsigned>(nfield));
  const int64_t* doff = pk.dev<int64_t>(o);
  if (vec) {
    if (skipna) ens_mean_kernel<4, true><<<grid, 256, 0, ctx->stream>>>(x, doff, out, nmember, member_stride, slab, nvec);
    else ens_mean_kernel<4, false><<<grid, 256, 0, ctx->stream>>>(x, doff, out, nmember, member_stride, slab, nvec);
  } else {
    if (skipna) ens_mean_kernel<1, true><<<grid, 256, 0, ctx->stream>>>(x, doff, out, nmember, member_stride, slab, nvec);
    else ens_mean_kernel<1, false><<<grid, 256, 0, ctx->stream>>>(x, doff, out, nmember, member_stride, slab, nvec);
  }
  WB2_CUDA_TRY(cudaGetLastError());
  ctx->launches += 1;
  WB2_TRY(pk.release());
  return WB2_OK;
}

extern "C" int wb2_spectrum_interp(wb2_ctx* ctx, const float* spec, int64_t nfield,
                                   int32_t nrow, int32_t nk, const double* freq_table,
                                   int32_t nfreq, const double* freqs, float* out) {
  WB2_NVTX("wb2_spectrum_interp");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_REQUIRE(nrow > 0 && nk >= 2 && nfreq > 0 && nfield >= 0, "bad sizes");
  if (nfield == 0) return WB2_OK;
  WB2_REQUIRE(spec && freq_table && freqs && out, "NULL argument");
  DeviceGuard guard(ctx->device);
  Packer pk(ctx);
  const size_t o1 = pk.add(freq_table, size_t(nrow) * nk * sizeof(double));
  const size_t o2 = pk.add(freqs, size_t(nfreq) * sizeof(double));
  WB2_TRY(pk.commit());
  const int64_t total = nfield * nrow * int64_t(nfreq);
  const int64_t blocks = std::min<int64_t>((total + 255) / 256, int64_t(ctx->num_sms) * 16);
  spectrum_interp_kernel<<<static_cast<unsigned>(blocks), 256, 0, ctx->stream>>>(
      spec, pk.dev<double>(o1), pk.dev<double>(o2), out, nfield, nrow, nk, nfreq);
  WB2_CUDA_TRY(cudaGetLastError());
  ctx->launches += 1;
  WB2_TRY(pk.release());
  return WB2_OK;
}

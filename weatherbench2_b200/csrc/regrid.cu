// K5 -- conservative lat/lon regridding (sm_90a).
//
// Replaces ConservativeRegridder.regrid_array = _nanmean
// (weatherbench2/regridding.py:502-536):
//     total = einsum('ab,cd,...bd->...ac', Wlon, Wlat, where(isnan(x), 0, x))
//     count = einsum('ab,cd,...bd->...ac', Wlon, Wlat, ~isnan(x))
//     out   = total / count                      (NaN where count == 0)
// The reference contracts with two DENSE matrices per 2-D slice inside a
// Python-level loop (xr.apply_ufunc(vectorize=True), regridding.py:198-205),
// although both matrices are banded (7 taps at 0.25 -> 1.5 degrees).  Here the
// weights arrive in CSR form and one CTA produces a group of G target
// longitudes of one field:
//   stage 1  every source row (longitude) the group touches is read ONCE from
//            HBM: thread d-strided over the contiguous source latitude, each
//            loaded value feeds the G register accumulators
//            y_a[d] += Wlon[a,b] x0[b,d],  v_a[d] += Wlon[a,b] valid[b,d]
//            (dense G-wide table of the group's weights in shared memory, rows
//            unrolled 4x so 12 independent loads are in flight per thread);
//   stage 2  out[a,c] = (sum_d Wlat[c,d] y_a[d]) / (sum_d Wlat[c,d] v_a[d])
//            from shared memory.
// Arithmetic is float32 like the reference (JAX default); the order of
// summation differs (taps in ascending source index).  Target cells the source
// grid does not cover (NaN weight rows, regridding.py:367-371, 493-497) are NaN.
// Banded semantics: a target cell sees only its own taps, so +-inf reach only
// the cells whose footprint holds them (the reference's dense contraction
// multiplies them by zero weights and turns the whole slice NaN).
//
// Roofline: HBM, 4 B read per source cell + 4 B written per target cell.
#include <algorithm>

#include "common.cuh"

namespace wb2 {

constexpr int kRgThreads = 256;
constexpr int kRgGroup = 4;  // target longitudes per CTA
constexpr int kRgMaxDpt = 4;  // source latitudes per thread (<= 1024 latitudes)

struct RegridParams {
  const float* src;
  float* dst;
  int64_t src_field_stride, dst_field_stride;
  const int32_t* grp_rows;  // [ngroups][maxnb] source rows of the group (-1 pad)
  const float* grp_w;       // [ngroups][maxnb][kRgGroup]
  const int32_t* grp_nb;    // [ngroups]
  const int32_t* lon_ptr;   // [nlon_t + 1] the longitude CSR, for the columns
  const int32_t* lon_idx;   //   that hold a NaN or an infinity
  const float* lon_val;
  const uint8_t* lon_nan;   // [nlon_t]
  const int32_t* lat_ptr;   // [nlat_t + 1]
  const int32_t* lat_idx;
  const float* lat_val;
  const uint8_t* lat_nan;  // [nlat_t]
  int32_t nlon_s, nlat_s, nlon_t, nlat_t;
  int32_t ngroups, maxnb;
};

// Column d of a group whose accumulation met a NaN or an infinity: y and v of
// each target over its OWN taps, in CSR order, NaN as missing (out of line, so
// that the hot loop keeps its registers).
__device__ __noinline__ void regrid_own_taps(const float* __restrict__ x, int d, int nlat_s,
                                             const int32_t* __restrict__ ptr, int na,
                                             const int32_t* __restrict__ idx,
                                             const float* __restrict__ val, float* ybuf) {
  for (int a = 0; a < na; ++a) {
    float yy = 0.f, vv = 0.f;
    const int t1 = __ldg(ptr + a + 1);
    for (int tp = __ldg(ptr + a); tp < t1; ++tp) {
      const float w = __ldg(val + tp);
      const float xq = __ldg(x + int64_t(__ldg(idx + tp)) * nlat_s + d);
      const bool ok = xq == xq;
      yy = fmaf(w, ok ? xq : 0.f, yy);
      vv = fmaf(w, ok ? 1.f : 0.f, vv);
    }
    ybuf[(a * 2 + 0) * nlat_s + d] = yy;
    ybuf[(a * 2 + 1) * nlat_s + d] = vv;
  }
}

template <int kRgDpt>
__global__ void __launch_bounds__(kRgThreads) regrid_kernel(const RegridParams p) {
  extern __shared__ __align__(16) float sm[];
  float* ybuf = sm;                                         // [G][2][nlat_s]
  float* wtab = sm + size_t(kRgGroup) * 2 * p.nlat_s;       // [maxnb][G]
  int* rows = reinterpret_cast<int*>(wtab + size_t(p.maxnb) * kRgGroup);  // [maxnb]

  const int64_t field = blockIdx.x / p.ngroups;
  const int g = blockIdx.x % p.ngroups;
  const int a0 = g * kRgGroup;
  const int na = min(kRgGroup, p.nlon_t - a0);
  const int nb = p.grp_nb[g];
  for (int i = threadIdx.x; i < nb * kRgGroup; i += kRgThreads)
    wtab[i] = p.grp_w[size_t(g) * p.maxnb * kRgGroup + i];
  for (int i = threadIdx.x; i < nb; i += kRgThreads) rows[i] = p.grp_rows[size_t(g) * p.maxnb + i];
  __syncthreads();
  float* s_wsum = reinterpret_cast<float*>(rows + p.maxnb);  // [G] weight row sums
  if (threadIdx.x < kRgGroup) {
    float ws = 0.f;
    for (int bi = 0; bi < nb; ++bi) ws = fmaf(wtab[bi * kRgGroup + threadIdx.x], 1.f, ws);
    s_wsum[threadIdx.x] = ws;
  }
  __syncthreads();

  const float* __restrict__ x = p.src + field * p.src_field_stride;
  const float nanv = __int_as_float(0x7fc00000);

  // ---- stage 1: contract over source longitude, every source row read once ---
  // The valid-weight sum v = sum_b W[a,b] [x[b,d] not NaN] equals the plain row
  // sum of the weights unless a NaN is met, so the hot loop only accumulates
  // y = sum_b W[a,b] x[b,d] WITHOUT looking at the values: a NaN or an infinity
  // anywhere in the column makes some y of the group NaN or infinite (the dense
  // table's zeros give 0 * inf = NaN).  Those columns recompute y and v over
  // each target's OWN taps (second pass over the same rows, served by L1/L2),
  // so a target sees only its own taps, exactly as in regrid_tma_kernel.
  const float infv = __int_as_float(0x7f800000);
  float y[kRgDpt][kRgGroup];
#pragma unroll
  for (int i = 0; i < kRgDpt; ++i) {
#pragma unroll
    for (int a = 0; a < kRgGroup; ++a) y[i][a] = 0.f;
  }

#pragma unroll 4
  for (int bi = 0; bi < nb; ++bi) {
    const float* __restrict__ row = x + int64_t(rows[bi]) * p.nlat_s;
    float xv[kRgDpt];
#pragma unroll
    for (int i = 0; i < kRgDpt; ++i) {
      const int d = threadIdx.x + i * kRgThreads;
      xv[i] = d < p.nlat_s ? __ldg(row + d) : 0.f;
    }
    const float4 w4 = *reinterpret_cast<const float4*>(wtab + bi * kRgGroup);
    const float w[kRgGroup] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
    for (int i = 0; i < kRgDpt; ++i)
#pragma unroll
      for (int a = 0; a < kRgGroup; ++a) y[i][a] = fmaf(w[a], xv[i], y[i][a]);
  }
  // v for finite columns: the weights' row sums, added in the same order and
  // rounding as the explicit accumulation would (bit-identical)
  float wsum[kRgGroup];
#pragma unroll
  for (int a = 0; a < kRgGroup; ++a) wsum[a] = s_wsum[a];
#pragma unroll
  for (int i = 0; i < kRgDpt; ++i) {
    const int d = threadIdx.x + i * kRgThreads;
    if (d < p.nlat_s) {
      bool bad = false;
#pragma unroll
      for (int a = 0; a < kRgGroup; ++a) {
        bad |= !(fabsf(y[i][a]) < infv);
        ybuf[(a * 2 + 0) * p.nlat_s + d] = y[i][a];
        ybuf[(a * 2 + 1) * p.nlat_s + d] = wsum[a];
      }
      if (bad)
        regrid_own_taps(x, d, p.nlat_s, p.lon_ptr + a0, na, p.lon_idx, p.lon_val, ybuf);
    }
  }
  __syncthreads();

  // ---- stage 2: contract over source latitude, divide, store ----------------
  float* out = p.dst + field * p.dst_field_stride;
  const int nout = na * p.nlat_t;
  for (int o = threadIdx.x; o < nout; o += kRgThreads) {
    const int al = o / p.nlat_t;
    const int c = o - al * p.nlat_t;
    float r;
    if (p.lon_nan[a0 + al] || p.lat_nan[c]) {
      r = nanv;
    } else {
      const float* yy = ybuf + size_t(al) * 2 * p.nlat_s;
      const float* vv = yy + p.nlat_s;
      float tot = 0.f, cnt = 0.f;
      const int t0 = p.lat_ptr[c], t1 = p.lat_ptr[c + 1];
      for (int tp = t0; tp < t1; ++tp) {
        const float w = p.lat_val[tp];
        const int d = p.lat_idx[tp];
        tot = fmaf(w, yy[d], tot);
        cnt = fmaf(w, vv[d], cnt);
      }
      r = tot / cnt;  // 0 / 0 -> NaN on purpose (regridding.py:534)
    }
    out[int64_t(a0 + al) * p.nlat_t + c] = r;
  }
}

static int check_csr(const wb2_csr* m, const char* name) {
  WB2_REQUIRE(m != nullptr, "%s weights are NULL", name);
  WB2_REQUIRE(m->n_src > 0 && m->n_tgt > 0, "%s: empty axis", name);
  WB2_REQUIRE(m->row_ptr && m->col_idx && m->val && m->nan_row, "%s: NULL CSR arrays", name);
  WB2_REQUIRE(m->row_ptr[0] == 0, "%s: row_ptr[0] must be 0", name);
  for (int i = 0; i < m->n_tgt; ++i)
    WB2_REQUIRE(m->row_ptr[i + 1] >= m->row_ptr[i], "%s: row_ptr must be non-decreasing", name);
  const int nnz = m->row_ptr[m->n_tgt];
  for (int i = 0; i < nnz; ++i)
    WB2_REQUIRE(m->col_idx[i] >= 0 && m->col_idx[i] < m->n_src, "%s: col_idx out of range",
                name);
  // Both kernels add a target's taps in ascending source order; the TMA kernel
  // walks the CSR as given and this one the sorted union of a group's rows, so
  // they agree only when every row is sorted and free of duplicates.
  for (int i = 0; i < m->n_tgt; ++i)
    for (int tp = m->row_ptr[i] + 1; tp < m->row_ptr[i + 1]; ++tp)
      WB2_REQUIRE(m->col_idx[tp] > m->col_idx[tp - 1],
                  "%s: col_idx must be strictly increasing within a row (row %d)", name, i);
  return WB2_OK;
}

// regrid_tma.cu: TMA-staged persistent variant (1 = handled, 0 = not eligible)
int regrid_tma_try(wb2_ctx* ctx, const float* src, float* dst, int64_t nfield,
                   int64_t src_field_stride, int64_t dst_field_stride, const wb2_csr* lon_w,
                   const wb2_csr* lat_w);

}  // namespace wb2

using namespace wb2;

extern "C" int wb2_regrid_conservative(wb2_ctx* ctx, const float* src, float* dst,
                                       int64_t nfield, int64_t src_field_stride,
                                       int64_t dst_field_stride, const wb2_csr* lon_w,
                                       const wb2_csr* lat_w) {
  WB2_NVTX("wb2_regrid_conservative");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_TRY(check_csr(lon_w, "longitude"));
  WB2_TRY(check_csr(lat_w, "latitude"));
  WB2_REQUIRE(nfield >= 0 && nfield <= (int64_t(1) << 24), "nfield out of range");
  if (nfield == 0) return WB2_OK;
  WB2_REQUIRE(src && dst, "src/dst are NULL");
  WB2_REQUIRE(src_field_stride >= int64_t(lon_w->n_src) * lat_w->n_src,
              "src_field_stride smaller than a source slab");
  WB2_REQUIRE(dst_field_stride >= int64_t(lon_w->n_tgt) * lat_w->n_tgt,
              "dst_field_stride smaller than a target slab");
  if (lat_w->n_src > kRgThreads * kRgMaxDpt) {
    set_error("wb2_regrid_conservative: at most %d source latitudes are supported (got %d)",
              kRgThreads * kRgMaxDpt, lat_w->n_src);
    return WB2_EUNSUPPORTED;
  }
  DeviceGuard guard(ctx->device);
  {
    const int trc = regrid_tma_try(ctx, src, dst, nfield, src_field_stride, dst_field_stride,
                                   lon_w, lat_w);
    if (trc != 0) return trc < 0 ? trc : WB2_OK;
  }

  // per-group union of source rows + dense G-wide weight table (host, tiny)
  const int nlon_t = lon_w->n_tgt;
  const int ngroups = (nlon_t + kRgGroup - 1) / kRgGroup;
  std::vector<std::vector<int>> grows(ngroups);
  int maxnb = 1;
  for (int g = 0; g < ngroups; ++g) {
    std::vector<int>& r = grows[g];
    for (int a = g * kRgGroup; a < std::min(nlon_t, (g + 1) * kRgGroup); ++a)
      for (int tp = lon_w->row_ptr[a]; tp < lon_w->row_ptr[a + 1]; ++tp)
        r.push_back(lon_w->col_idx[tp]);
    std::sort(r.begin(), r.end());
    r.erase(std::unique(r.begin(), r.end()), r.end());
    maxnb = std::max<int>(maxnb, static_cast<int>(r.size()));
  }
  std::vector<int32_t> h_rows(size_t(ngroups) * maxnb, 0);
  std::vector<float> h_w(size_t(ngroups) * maxnb * kRgGroup, 0.f);
  std::vector<int32_t> h_nb(ngroups, 0);
  for (int g = 0; g < ngroups; ++g) {
    const std::vector<int>& r = grows[g];
    h_nb[g] = static_cast<int>(r.size());
    for (size_t bi = 0; bi < r.size(); ++bi) h_rows[size_t(g) * maxnb + bi] = r[bi];
    for (int a = g * kRgGroup; a < std::min(nlon_t, (g + 1) * kRgGroup); ++a)
      for (int tp = lon_w->row_ptr[a]; tp < lon_w->row_ptr[a + 1]; ++tp) {
        const size_t bi = std::lower_bound(r.begin(), r.end(), lon_w->col_idx[tp]) - r.begin();
        h_w[(size_t(g) * maxnb + bi) * kRgGroup + (a - g * kRgGroup)] = lon_w->val[tp];
      }
  }

  const int nlat_nnz = lat_w->row_ptr[lat_w->n_tgt] > 0 ? lat_w->row_ptr[lat_w->n_tgt] : 1;
  const int nlon_nnz = std::max(1, lon_w->row_ptr[nlon_t]);
  Packer pk(ctx);
  size_t o1 = pk.add(h_rows.data(), h_rows.size() * 4);
  size_t o2 = pk.add(h_w.data(), h_w.size() * 4);
  size_t o3 = pk.add(h_nb.data(), h_nb.size() * 4);
  size_t o9 = pk.add(lon_w->row_ptr, size_t(nlon_t + 1) * 4);
  size_t o10 = pk.add(lon_w->col_idx, size_t(nlon_nnz) * 4);
  size_t o11 = pk.add(lon_w->val, size_t(nlon_nnz) * 4);
  size_t o4 = pk.add(lon_w->nan_row, size_t(lon_w->n_tgt));
  size_t o5 = pk.add(lat_w->row_ptr, size_t(lat_w->n_tgt + 1) * 4);
  size_t o6 = pk.add(lat_w->col_idx, size_t(nlat_nnz) * 4);
  size_t o7 = pk.add(lat_w->val, size_t(nlat_nnz) * 4);
  size_t o8 = pk.add(lat_w->nan_row, size_t(lat_w->n_tgt));
  WB2_TRY(pk.commit());

  RegridParams p;
  p.src = src; p.dst = dst;
  p.src_field_stride = src_field_stride; p.dst_field_stride = dst_field_stride;
  p.grp_rows = pk.dev<int32_t>(o1); p.grp_w = pk.dev<float>(o2);
  p.grp_nb = pk.dev<int32_t>(o3); p.lon_nan = pk.dev<uint8_t>(o4);
  p.lon_ptr = pk.dev<int32_t>(o9); p.lon_idx = pk.dev<int32_t>(o10);
  p.lon_val = pk.dev<float>(o11);
  p.lat_ptr = pk.dev<int32_t>(o5); p.lat_idx = pk.dev<int32_t>(o6);
  p.lat_val = pk.dev<float>(o7); p.lat_nan = pk.dev<uint8_t>(o8);
  p.nlon_s = lon_w->n_src; p.nlat_s = lat_w->n_src;
  p.nlon_t = lon_w->n_tgt; p.nlat_t = lat_w->n_tgt;
  p.ngroups = ngroups; p.maxnb = maxnb;
  const size_t smem = (size_t(kRgGroup) * 2 * p.nlat_s + size_t(maxnb) * kRgGroup) * sizeof(float) +
                      size_t(maxnb) * sizeof(int) + kRgGroup * sizeof(float);
  WB2_REQUIRE(smem <= 200 * 1024, "wb2_regrid_conservative: weights too dense for shared memory");
  const int dpt = (p.nlat_s + kRgThreads - 1) / kRgThreads;
  auto go = [&](auto kernel) -> int {
    if (smem > 48 * 1024)
      WB2_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        static_cast<int>(smem)));
    kernel<<<static_cast<unsigned>(nfield * ngroups), kRgThreads, smem, ctx->stream>>>(p);
    WB2_CUDA_TRY(cudaGetLastError());
    return WB2_OK;
  };
  int rc;
  switch (dpt) {
    case 1: rc = go(regrid_kernel<1>); break;
    case 2: rc = go(regrid_kernel<2>); break;
    case 3: rc = go(regrid_kernel<3>); break;
    default: rc = go(regrid_kernel<4>); break;
  }
  if (rc != WB2_OK) return rc;
  ctx->launches += 1;
  WB2_TRY(pk.release());
  return WB2_OK;
}

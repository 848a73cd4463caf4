// K3 -- energy-score sums (sm_90a).
//
// EnergyScoreSkill  = mean_m sqrt(SA((x_m - t)^2))           (metrics.py:1503-1517)
// EnergyScoreSpread = mean_{m<M-1} sqrt(SA((x_m - x_{m+1})^2)) (metrics.py:1471-1496)
// need 2M - 1 weighted spatial sums per field.  The reference materialises an
// M-sized difference array for each; running K1 once per member pair reads the
// ensemble ~4 times from HBM.  Here the members are split into groups of GS
// consecutive members, one warp per (row, group): a lane owns a grid point,
// loads its GS (+1 for the pair that straddles the group edge) members with all
// loads in flight, and keeps only 2 GS + 1 accumulators, so occupancy stays
// high.  HBM sees every member once; the straddling member and the truth are
// re-read through L1/L2 by the neighbouring warp of the same CTA.
// Per (row, segment): butterfly, then lane r applies region r's float64 weight.
//
// Roofline: (4 M + 4) bytes per grid point, ~4 FP32 instructions per member:
// HBM-bound.  NaN propagates (skipna = False only; the skipna path keeps using
// K1 on member views).
#include <algorithm>

#include "region_reduce.cuh"

namespace wb2 {

struct EsParams {
  const float* x;
  const float* t;
  const int64_t* off_x;
  const int64_t* off_t;
  const double* row_w;
  const int32_t* seg_start;
  const double* seg_w;
  const float* col_w;
  const float* cell_w;
  double* partial;  // [nfield][nblk][ngroups][R][2 * GS + 1]
  int64_t member_stride, row_stride;
  int32_t nmember, nrow, ncol, nregion, nseg, zero_skip, rows_per_block, nblk;
  int32_t ngroups;         // ceil(nmember / GS)
  int32_t rows_in_flight;  // warps per CTA / ngroups
  int32_t vec4;            // 1: every slab / segment is 16-byte aligned
};

// blockDim = 32 * ngroups * rows_in_flight; warp -> (row slot, member group)
template <int GS>
__global__ void __launch_bounds__(256, 2) energy_kernel(const EsParams p) {
  constexpr int NACC = 2 * GS + 1;  // skill[GS], spread[GS], weight sum
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* s_colw = reinterpret_cast<float*>(smem_raw);

  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int group = warp % p.ngroups;
  const int slot = warp / p.ngroups;
  const int64_t field = blockIdx.x / p.nblk;
  const int blk = blockIdx.x % p.nblk;
  const int R = p.nregion;
  const int M = p.nmember;
  const int m0 = group * GS;
  const bool weighted = p.col_w != nullptr || p.cell_w != nullptr;
  if (p.col_w) {
    for (int i = threadIdx.x; i < p.ncol; i += blockDim.x) s_colw[i] = p.col_w[i];
    __syncthreads();
  }
  const float* __restrict__ px = p.x + p.off_x[field] + int64_t(m0) * p.member_stride;
  const float* __restrict__ pt = p.t + p.off_t[field];
  const bool zero_skip = p.zero_skip != 0;

  double accd[NACC];
#pragma unroll
  for (int i = 0; i < NACC; ++i) accd[i] = 0.0;

  const int row0 = blk * p.rows_per_block;
  const int row1 = min(p.nrow, row0 + p.rows_per_block);
  for (int row = row0 + slot; row < row1; row += p.rows_in_flight) {
    const int64_t rbase = int64_t(row) * p.row_stride;
    for (int k = 0; k < p.nseg; ++k) {
      const int s = p.seg_start[k];
      const int e = p.seg_start[k + 1];
      float acc[NACC];
#pragma unroll
      for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
      int col_begin = s + lane;
      if (p.vec4 && !weighted) {
        // 128-bit loads: a lane owns 4 consecutive columns, so four times the
        // bytes are in flight per load instruction (scalar loads leave this
        // kernel latency-bound).  Host guarantees 16-byte alignment and
        // (e - s) % 4 == 0.
        for (int col = s + lane * 4; col < e; col += 128) {
          const float* src = px + rbase + col;
          const float4 t4 = ldg_stream(reinterpret_cast<const float4*>(pt + rbase + col));
          float4 v[GS + 1];
#pragma unroll
          for (int j = 0; j <= GS; ++j)
            v[j] = (m0 + j) < M
                       ? ldg_stream(reinterpret_cast<const float4*>(src + int64_t(j) * p.member_stride))
                       : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
          for (int j = 0; j < GS; ++j) {
            if (m0 + j < M) {
              const float d0 = v[j].x - t4.x, d1 = v[j].y - t4.y, d2 = v[j].z - t4.z,
                          d3 = v[j].w - t4.w;
              acc[j] += (d0 * d0 + d1 * d1) + (d2 * d2 + d3 * d3);
              if (m0 + j + 1 < M) {
                const float g0 = v[j].x - v[j + 1].x, g1 = v[j].y - v[j + 1].y,
                            g2 = v[j].z - v[j + 1].z, g3 = v[j].w - v[j + 1].w;
                acc[GS + j] += (g0 * g0 + g1 * g1) + (g2 * g2 + g3 * g3);
              }
            }
          }
          acc[2 * GS] += 4.f;
        }
        col_begin = e;  // nothing left for the scalar loop
      }
      for (int col = col_begin; col < e; col += 32) {
        float wc = 1.f;
        if (weighted) {
          if (p.col_w) wc *= s_colw[col];
          if (p.cell_w) wc *= p.cell_w[int64_t(row) * p.ncol + col];
          if (zero_skip && wc == 0.f) continue;
        }
        const float* src = px + rbase + col;
        const float t = __ldg(pt + rbase + col);
        float v[GS + 1];
#pragma unroll
        for (int j = 0; j <= GS; ++j)
          v[j] = (m0 + j) < M ? __ldg(src + int64_t(j) * p.member_stride) : 0.f;
#pragma unroll
        for (int j = 0; j < GS; ++j) {
          if (m0 + j < M) {
            const float d = v[j] - t;
            acc[j] = fmaf(weighted ? wc * d : d, d, acc[j]);
            if (m0 + j + 1 < M) {
              const float g = v[j] - v[j + 1];
              acc[GS + j] = fmaf(weighted ? wc * g : g, g, acc[GS + j]);
            }
          }
        }
        acc[2 * GS] += wc;
      }
#pragma unroll
      for (int i = 0; i < NACC; ++i) acc[i] = warp_sum(acc[i]);
      if (lane < R) {
        const double w = p.row_w[int64_t(lane) * p.nrow + row] * p.seg_w[lane * p.nseg + k];
        if (!(zero_skip && w == 0.0)) {
#pragma unroll
          for (int i = 0; i < NACC; ++i) accd[i] += w * double(acc[i]);
        }
      }
    }
  }
  // per-(CTA, row slot, group) partials; the finalize kernel adds the slots
  if (lane < R) {
    double* out = p.partial +
                  ((((field * p.nblk + blk) * p.rows_in_flight + slot) * p.ngroups + group) *
                       int64_t(R) + lane) * NACC;
#pragma unroll
    for (int i = 0; i < NACC; ++i) out[i] = accd[i];
  }
}

// partial [nfield][nblk][slots][ngroups][R][2*GS+1] -> out [nfield][R][4][M]
__global__ void energy_finalize_kernel(const double* __restrict__ partial,
                                       double* __restrict__ out, int nblk, int slots,
                                       int ngroups, int R, int GS, int M) {
  const int64_t field = blockIdx.x;
  const int nacc = 2 * GS + 1;
  for (int idx = threadIdx.x; idx < R * 4 * M; idx += blockDim.x) {
    const int r = idx / (4 * M);
    const int q = (idx / M) % 4;
    const int m = idx % M;
    const int g = m / GS, j = m % GS;
    int src = -1;
    if (q == 0) src = j;
    else if (q == 1) src = m < M - 1 ? GS + j : -1;
    else src = (q == 3 && m >= M - 1) ? -1 : 2 * GS;  // weight sums
    double v = 0.0;
    if (src >= 0)
      for (int b = 0; b < nblk * slots; ++b)
        v += partial[(((field * nblk * slots + b) * ngroups + g) * int64_t(R) + r) * nacc + src];
    out[field * int64_t(R) * 4 * M + idx] = v;
  }
}

}  // namespace wb2

using namespace wb2;

extern "C" int wb2_energy_score(wb2_ctx* ctx, const void* x, const void* t, int dtype,
                                int32_t nmember, int64_t member_stride, int64_t nfield,
                                const int64_t* off_x, const int64_t* off_t,
                                const wb2_weights* w, double* out) {
  WB2_NVTX("wb2_energy_score");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_REQUIRE(dtype == WB2_F32, "wb2_energy_score: only WB2_F32 inputs are supported");
  WB2_REQUIRE(nmember >= 1 && nmember <= 64,
              "wb2_energy_score: 1..64 ensemble members are supported (got %d)", nmember);
  WB2_TRY(validate_weights(w));
  WB2_REQUIRE(out != nullptr, "out is NULL");
  WB2_REQUIRE(nfield >= 0 && nfield <= (int64_t(1) << 24), "nfield out of range");
  if (nfield == 0) return WB2_OK;
  WB2_REQUIRE(x && t && off_x && off_t, "x/t and their offset tables must not be NULL");
  DeviceGuard guard(ctx->device);

  const int gs = nmember <= 4 ? 4 : 8;
  const int ngroups = (nmember + gs - 1) / gs;  // <= 8
  const int rows_in_flight = std::max(1, 8 / ngroups);
  const int warps = ngroups * rows_in_flight;
  const BlockRows br =
      block_rows(w->nrow, nfield, 8 * rows_in_flight, rows_in_flight, 4 * ctx->num_sms);
  const int nblk = br.nblk;
  const int R = w->nregion;
  const int nacc = 2 * gs + 1;
  Packer pk(ctx);
  size_t o_x = pk.add(off_x, nfield * sizeof(int64_t));
  size_t o_t = pk.add(off_t, nfield * sizeof(int64_t));
  const WeightUpload wu(pk, w);
  size_t o_part = pk.reserve(size_t(nfield) * nblk * rows_in_flight * ngroups * R * nacc *
                             sizeof(double));
  WB2_TRY(pk.commit());
  EsParams p;
  p.x = static_cast<const float*>(x);
  p.t = static_cast<const float*>(t);
  p.off_x = pk.dev<int64_t>(o_x); p.off_t = pk.dev<int64_t>(o_t);
  wu.bind(p);
  p.partial = pk.dev<double>(o_part);
  p.member_stride = member_stride;
  p.nmember = nmember;
  p.rows_per_block = br.rows_per_block; p.nblk = nblk;
  p.ngroups = ngroups; p.rows_in_flight = rows_in_flight;
  {
    bool ok = (reinterpret_cast<uintptr_t>(x) & 15) == 0 &&
              (reinterpret_cast<uintptr_t>(t) & 15) == 0 && member_stride % 4 == 0 &&
              w->row_stride % 4 == 0;
    for (int k = 0; k <= w->nseg && ok; ++k) ok = w->seg_start[k] % 4 == 0;
    for (int64_t i = 0; i < nfield && ok; ++i) ok = off_x[i] % 4 == 0 && off_t[i] % 4 == 0;
    p.vec4 = ok ? 1 : 0;
  }
  const size_t smem = w->col_w ? size_t(w->ncol) * sizeof(float) : 0;
  WB2_TRY(launch_kernel(ctx, gs == 4 ? energy_kernel<4> : energy_kernel<8>,
                        dim3(static_cast<unsigned>(nfield * nblk)), 32 * warps, smem, p));
  energy_finalize_kernel<<<static_cast<unsigned>(nfield), 128, 0, ctx->stream>>>(
      p.partial, out, nblk, rows_in_flight, ngroups, R, gs, nmember);
  WB2_CUDA_TRY(cudaGetLastError());
  ctx->launches += 2;
  WB2_TRY(pk.release());
  return WB2_OK;
}

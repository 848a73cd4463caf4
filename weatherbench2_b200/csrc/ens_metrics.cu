// K2 -- fused ensemble metrics (sm_90a).
//
// One read of the M members (+ truth) of every grid point yields the five
// point-wise quantities behind CRPS / CRPSSkill / CRPSSpread
// (weatherbench2/metrics.py:657-715, 781-846), EnsembleMeanMSE / RMSE
// (:1293-1333), EnsembleVariance / Stddev (:1185-1241) and
// DebiasedEnsembleMeanMSE (:532-565, :1347-1363), which are then reduced over
// latitude x longitude with the same weight machinery as K1:
//   [0] skill_pt  = mean_m |t - x_m|                          (metrics.py:824)
//   [1] spread_pt = 2 * mean_m((2 r_m - M - 1) x_m) / (M - 1) (metrics.py:805-813)
//   [2] (t - xbar)^2          [3] var_m(x, ddof=1)     [4] [2] - [3] / M
// The reference ranks with np.argsort + put_along_axis on an int64 copy of the
// whole ensemble (:836-846); here the members of a point sit in registers and
// go through a Batcher sorting network (sort_networks.inc), after which
// sum_i (2 i - M - 1) x_(i) is the same quantity (ties do not matter).
//
// Roofline: (4 M + 4) bytes per grid point from HBM; the sorting network is
// ~2 * 403 FMNMX per point at M = 50, which puts this kernel near the
// ALU-pipe / HBM ridge (see DESIGN.md).
#include <cmath>

#include "region_reduce.cuh"
#include "ens_point.cuh"

namespace wb2 {

constexpr int kEnsWarps = 4;
constexpr int kEnsThreads = kEnsWarps * 32;

struct EnsParams {
  const float* x;
  const float* t;
  const int64_t* off_x;
  const int64_t* off_t;
  const double* row_w;       // [R][nrow]
  const int32_t* seg_start;  // [nseg + 1]
  const double* seg_w;       // [R][nseg]
  const float* col_w;        // [ncol] or null
  const float* cell_w;       // [nrow][ncol] or null
  double* partial;           // [nfield][nblk][R][WB2_ENS_NSTAT]
  int64_t member_stride;
  int64_t row_stride;
  int32_t nmember;
  int32_t nrow, ncol;
  int32_t nregion, nseg;
  int32_t zero_skip;
  int32_t rows_per_block;
  int32_t nblk;
};

// resident CTAs per SM the register allocation targets: 4 with skipna, 5 without
template <int MP, bool SKIPNA, bool EXACT, bool TWIN = false>
__global__ void __launch_bounds__(kEnsThreads, SKIPNA ? 4 : 5)
    ens_metrics_kernel(const EnsParams p) {
  constexpr int NCNT = SKIPNA ? kEnsStats : 1;
  constexpr int NS = kEnsStats + NCNT;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double* red = reinterpret_cast<double*>(smem_raw);                    // [warps][32][NS]
  float* s_colw = reinterpret_cast<float*>(red + kEnsWarps * 32 * NS);  // [ncol]

  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int64_t field = blockIdx.x / p.nblk;
  const int blk = blockIdx.x % p.nblk;
  const int R = p.nregion;
  const int M = p.nmember;
  const bool weighted = p.col_w != nullptr || p.cell_w != nullptr;
  if (p.col_w) {
    for (int i = threadIdx.x; i < p.ncol; i += kEnsThreads) s_colw[i] = p.col_w[i];
    __syncthreads();
  }
  const float* __restrict__ px = p.x + p.off_x[field];
  const float* __restrict__ pt = p.t + p.off_t[field];
  const bool zero_skip = p.zero_skip != 0;

  double accd[NS];
#pragma unroll
  for (int i = 0; i < NS; ++i) accd[i] = 0.0;

  const int row0 = blk * p.rows_per_block;
  const int row1 = min(p.nrow, row0 + p.rows_per_block);
  for (int row = row0 + warp; row < row1; row += kEnsWarps) {
    const int64_t rbase = int64_t(row) * p.row_stride;
    for (int k = 0; k < p.nseg; ++k) {
      const int s = p.seg_start[k];
      const int e = p.seg_start[k + 1];
      float acc[NS];
#pragma unroll
      for (int i = 0; i < NS; ++i) acc[i] = 0.f;
      for (int col = s + lane; col < e; col += 32) {
        float v[MP];
        const float* src = px + rbase + col;
#pragma unroll
        for (int m = 0; m < MP; ++m) {
          if (EXACT || m < M) v[m] = ldg_stream(src + int64_t(m) * p.member_stride);
          else v[m] = 0.f;
        }
        const float t = ldg_stream(pt + rbase + col);
        float wc = 1.f;
        if (weighted) {
          if (p.col_w) wc *= s_colw[col];
          if (p.cell_w) wc *= p.cell_w[int64_t(row) * p.ncol + col];
          if (zero_skip && wc == 0.f) continue;  // metrics.py:160
        }
        float val[kEnsStats];
        ens_point<MP, SKIPNA, EXACT, TWIN>(v, t, M, val);
#pragma unroll
        for (int i = 0; i < kEnsStats; ++i) {
          if (SKIPNA) {
            if (val[i] == val[i]) {
              acc[i] += wc * val[i];
              acc[kEnsStats + i] += wc;
            }
          } else {
            acc[i] += wc * val[i];
          }
        }
        if (!SKIPNA) acc[kEnsStats] += wc;
      }
#pragma unroll
      for (int i = 0; i < NS; ++i) acc[i] = warp_sum(acc[i]);
      if (lane < R) {
        const double w = p.row_w[int64_t(lane) * p.nrow + row] * p.seg_w[lane * p.nseg + k];
        if (!(zero_skip && w == 0.0)) {
#pragma unroll
          for (int i = 0; i < NS; ++i) accd[i] += w * double(acc[i]);
        }
      }
    }
  }

#pragma unroll
  for (int i = 0; i < NS; ++i) red[(warp * 32 + lane) * NS + i] = accd[i];
  __syncthreads();
  double* out = p.partial + (field * p.nblk + blk) * int64_t(R) * WB2_ENS_NSTAT;
  for (int idx = threadIdx.x; idx < R * WB2_ENS_NSTAT; idx += kEnsThreads) {
    const int r = idx / WB2_ENS_NSTAT;
    const int st = idx % WB2_ENS_NSTAT;
    const int slot = st < kEnsStats ? st : kEnsStats + (SKIPNA ? st - kEnsStats : 0);
    double v = 0.0;
#pragma unroll
    for (int w = 0; w < kEnsWarps; ++w) v += red[(w * 32 + r) * NS + slot];
    out[idx] = v;
  }
}

// ---------------------------------------------------------------------------
// Pair variant: a lane owns TWO adjacent grid points and every quantity is a
// register pair (lane 0 / 1 of the pair = the two points), members loaded as
// LDG.64.  Per point this halves the loads and index arithmetic, and the
// network's comparators split between FMNMX (ALU pipe) and FADD (FMA pipe).
// Full even ensembles, no skipna, separable weights with one column segment
// (the global region); everything else takes ens_metrics_kernel.
// ---------------------------------------------------------------------------
__device__ __forceinline__ u64x2f ldg_stream2(const float* p) {
  float a, b;
  asm volatile("ld.global.nc.L1::no_allocate.v2.f32 {%0,%1}, [%2];" : "=f"(a), "=f"(b) : "l"(p));
  return pk2f(a, b);
}

template <int MP, int OCC>
__global__ void __launch_bounds__(kEnsThreads, OCC) ens_pair_kernel(const EnsParams p) {
  constexpr int NS = kEnsStats + 1;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double* red = reinterpret_cast<double*>(smem_raw);  // [warps][32][NS]
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int64_t field = blockIdx.x / p.nblk;
  const int blk = blockIdx.x % p.nblk;
  const int R = p.nregion;
  const float* __restrict__ px = p.x + p.off_x[field];
  const float* __restrict__ pt = p.t + p.off_t[field];
  const bool zero_skip = p.zero_skip != 0;
  const float nanf_ = __int_as_float(0x7fc00000);

  double accd[NS];
#pragma unroll
  for (int i = 0; i < NS; ++i) accd[i] = 0.0;
  const int row0 = blk * p.rows_per_block;
  const int row1 = min(p.nrow, row0 + p.rows_per_block);
  for (int row = row0 + warp; row < row1; row += kEnsWarps) {
    const int64_t rbase = int64_t(row) * p.row_stride;
    float acc[NS];
#pragma unroll
    for (int i = 0; i < NS; ++i) acc[i] = 0.f;
    for (int col = 2 * lane; col < p.ncol; col += 64) {
      u64x2f v[MP];
      const float* src = px + rbase + col;
#pragma unroll
      for (int m = 0; m < MP; ++m) v[m] = ldg_stream2(src + int64_t(m) * p.member_stride);
      const u64x2f t2 = ldg_stream2(pt + rbase + col);
      // sums of the members and of |t - x_m| (metrics.py:824)
      u64x2f sumx = 0ull;
      float sa0 = 0.f, sa1 = 0.f;
#pragma unroll
      for (int m = 0; m < MP; ++m) {
        sumx = add2f(sumx, v[m]);
        float d0, d1;
        unpk2f(sub2f(t2, v[m]), d0, d1);
        sa0 += fabsf(d0);
        sa1 += fabsf(d1);
      }
      float sx0, sx1, t0, t1;
      unpk2f(sumx, sx0, sx1);
      unpk2f(t2, t0, t1);
      // divisions by the constants M and M - 1 as multiplications by their
      // float reciprocals (the IEEE division is a ~15-instruction subroutine,
      // eight of them per pair; differs from it by <= 1 ulp)
      constexpr float inv_m = 1.f / float(MP), inv_m1 = 1.f / float(MP - 1);
      const float mean0 = sx0 * inv_m, mean1 = sx1 * inv_m;
      const u64x2f mean2 = pk2f(mean0, mean1);
      u64x2f ss = 0ull;
#pragma unroll
      for (int m = 0; m < MP; ++m) {
        v[m] = sub2f(v[m], mean2);  // mean-removed: the spread sum is shift-invariant
        ss = fma2f(v[m], v[m], ss);
      }
      SortNet<MP>::run(v);
      u64x2f s2 = 0ull;
#pragma unroll
      for (int i = 0; i < MP; ++i) {
        const float coef = float(2 * (i + 1) - MP - 1);  // 2 r - M - 1, r = i + 1
        s2 = fma2f(v[i], pk2f(coef, coef), s2);
      }
      float ss0, ss1, s0, s1;
      unpk2f(ss, ss0, ss1);
      unpk2f(s2, s0, s1);
      float val0[kEnsStats], val1[kEnsStats];
      {
        const float var = ss0 * inv_m1, dm = t0 - mean0, mse = dm * dm;
        val0[0] = sa0 * inv_m;
        val0[1] = sx0 == sx0 ? 2.f * (s0 * inv_m) * inv_m1 : nanf_;
        val0[2] = mse;
        val0[3] = var;
        val0[4] = mse - var * inv_m;
      }
      {
        const float var = ss1 * inv_m1, dm = t1 - mean1, mse = dm * dm;
        val1[0] = sa1 * inv_m;
        val1[1] = sx1 == sx1 ? 2.f * (s1 * inv_m) * inv_m1 : nanf_;
        val1[2] = mse;
        val1[3] = var;
        val1[4] = mse - var * inv_m;
      }
#pragma unroll
      for (int i = 0; i < kEnsStats; ++i) acc[i] += val0[i] + val1[i];
      acc[kEnsStats] += 2.f;
    }
#pragma unroll
    for (int i = 0; i < NS; ++i) acc[i] = warp_sum(acc[i]);
    if (lane < R) {
      const double w = p.row_w[int64_t(lane) * p.nrow + row] * p.seg_w[lane];
      if (!(zero_skip && w == 0.0)) {
#pragma unroll
        for (int i = 0; i < NS; ++i) accd[i] += w * double(acc[i]);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < NS; ++i) red[(warp * 32 + lane) * NS + i] = accd[i];
  __syncthreads();
  double* out = p.partial + (field * p.nblk + blk) * int64_t(R) * WB2_ENS_NSTAT;
  for (int idx = threadIdx.x; idx < R * WB2_ENS_NSTAT; idx += kEnsThreads) {
    const int r = idx / WB2_ENS_NSTAT;
    const int st = idx % WB2_ENS_NSTAT;
    const int slot = st < kEnsStats ? st : kEnsStats;
    double v = 0.0;
#pragma unroll
    for (int w = 0; w < kEnsWarps; ++w) v += red[(w * 32 + r) * NS + slot];
    out[idx] = v;
  }
}

template <int MP>
constexpr bool kPairOk = MP >= 8 && MP % 2 == 0;

// 1 = launched, 0 = not eligible
template <int MP>
static int try_pair(wb2_ctx* ctx, const EnsParams& p, int64_t nfield, bool skipna,
                    bool aligned) {
  if constexpr (!kPairOk<MP>) {
    return 0;
  } else {
    const char* env = getenv("WB2_ENS_PATH");
    if (env && strcmp(env, "scalar") == 0) return 0;
    if (skipna || p.nmember != MP || !aligned || p.nseg != 1 || p.col_w || p.cell_w ||
        (p.ncol & 1) || (p.row_stride & 1) || (p.member_stride & 1))
      return 0;
    const size_t smem = size_t(kEnsWarps) * 32 * (kEnsStats + 1) * sizeof(double);
    const dim3 grid(static_cast<unsigned>(nfield * p.nblk));
    // registers: 2 MP for the member pairs + ~40; CTAs of 4 warps
    constexpr int OCC = MP <= 10 ? 6 : (MP <= 20 ? 4 : (MP <= 50 ? 3 : 2));
    ens_pair_kernel<MP, OCC><<<grid, kEnsThreads, smem, ctx->stream>>>(p);
    WB2_CUDA_TRY(cudaGetLastError());
    return 1;
  }
}

template <int MP>
static int launch_ens(wb2_ctx* ctx, const EnsParams& p, int64_t nfield, bool skipna,
                      bool aligned8) {
  {
    const int prc = try_pair<MP>(ctx, p, nfield, skipna, aligned8);
    if (prc != 0) return prc < 0 ? prc : WB2_OK;
  }
  const bool exact = p.nmember == MP;
  const int ns = kEnsStats + (skipna ? kEnsStats : 1);
  const size_t smem = size_t(kEnsWarps) * 32 * ns * sizeof(double) +
                      (p.col_w ? size_t(p.ncol) * sizeof(float) : 0);
  const dim3 grid(static_cast<unsigned>(nfield * p.nblk));
  auto go = [&](auto kernel) { return launch_kernel(ctx, kernel, grid, kEnsThreads, smem, p); };
  // full even ensembles without NaN handling sort with the twin ((a + b) - lo)
  // network; WB2_ENS_SORT=exact keeps the pure min / max network
  if constexpr (kTwinSortOk<MP, false, true>) {
    const char* sort_env = getenv("WB2_ENS_SORT");
    if (exact && !skipna && !(sort_env && strcmp(sort_env, "exact") == 0))
      return go(ens_metrics_kernel<MP, false, true, true>);
  }
  if (skipna) return exact ? go(ens_metrics_kernel<MP, true, true>)
                           : go(ens_metrics_kernel<MP, true, false>);
  return exact ? go(ens_metrics_kernel<MP, false, true>)
               : go(ens_metrics_kernel<MP, false, false>);
}

}  // namespace wb2

using namespace wb2;

extern "C" int wb2_ens_metrics(wb2_ctx* ctx, const void* x, const void* t, int dtype,
                               int32_t nmember, int64_t member_stride, int64_t nfield,
                               const int64_t* off_x, const int64_t* off_t,
                               const wb2_weights* w, int skipna, double* out) {
  WB2_NVTX("wb2_ens_metrics");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_REQUIRE(dtype == WB2_F32, "wb2_ens_metrics: only WB2_F32 inputs are supported");
  WB2_REQUIRE(nmember >= 1, "wb2_ens_metrics: nmember must be >= 1");
  WB2_TRY(validate_weights(w));
  WB2_REQUIRE(out != nullptr, "out is NULL");
  WB2_REQUIRE(nfield >= 0 && nfield <= (int64_t(1) << 24), "nfield out of range");
  if (nfield == 0) return WB2_OK;
  WB2_REQUIRE(x && t && off_x && off_t, "x/t and their offset tables must not be NULL");
  DeviceGuard guard(ctx->device);
  if (nmember > 64)  // rank-by-counting path (ens_big.cu)
    return ens_metrics_big(ctx, static_cast<const float*>(x), static_cast<const float*>(t),
                           nmember, member_stride, nfield, off_x, off_t, w, skipna, out);

  const BlockRows br = block_rows(w->nrow, nfield, 2 * kEnsWarps, kEnsWarps, 4 * ctx->num_sms);
  const size_t per_field = size_t(w->nregion) * WB2_ENS_NSTAT;
  Packer pk(ctx);
  size_t o_x = pk.add(off_x, nfield * sizeof(int64_t));
  size_t o_t = pk.add(off_t, nfield * sizeof(int64_t));
  const WeightUpload wu(pk, w);
  size_t o_part = pk.reserve(size_t(nfield) * br.nblk * per_field * sizeof(double));
  WB2_TRY(pk.commit());

  EnsParams p;
  p.x = static_cast<const float*>(x);
  p.t = static_cast<const float*>(t);
  p.off_x = pk.dev<int64_t>(o_x);
  p.off_t = pk.dev<int64_t>(o_t);
  wu.bind(p);
  p.partial = pk.dev<double>(o_part);
  p.member_stride = member_stride;
  p.nmember = nmember;
  p.rows_per_block = br.rows_per_block; p.nblk = br.nblk;

  int rc;
  const bool sk = skipna != 0;
  // the pair kernel reads two adjacent points with one 64-bit load
  bool aligned8 = (reinterpret_cast<uintptr_t>(x) & 7) == 0 &&
                  (reinterpret_cast<uintptr_t>(t) & 7) == 0;
  for (int64_t i = 0; aligned8 && i < nfield; ++i)
    aligned8 = ((off_x[i] | off_t[i]) & 1) == 0;
  if (nmember <= 2) rc = launch_ens<2>(ctx, p, nfield, sk, aligned8);
  else if (nmember <= 3) rc = launch_ens<3>(ctx, p, nfield, sk, aligned8);
  else if (nmember <= 4) rc = launch_ens<4>(ctx, p, nfield, sk, aligned8);
  else if (nmember <= 5) rc = launch_ens<5>(ctx, p, nfield, sk, aligned8);
  else if (nmember <= 8) rc = launch_ens<8>(ctx, p, nfield, sk, aligned8);
  else if (nmember <= 10) rc = launch_ens<10>(ctx, p, nfield, sk, aligned8);
  else if (nmember <= 16) rc = launch_ens<16>(ctx, p, nfield, sk, aligned8);
  else if (nmember <= 20) rc = launch_ens<20>(ctx, p, nfield, sk, aligned8);
  else if (nmember <= 32) rc = launch_ens<32>(ctx, p, nfield, sk, aligned8);
  else if (nmember <= 50) rc = launch_ens<50>(ctx, p, nfield, sk, aligned8);
  else rc = launch_ens<64>(ctx, p, nfield, sk, aligned8);
  if (rc != WB2_OK) return rc;
  WB2_TRY(launch_block_sum(ctx, p.partial, out, nfield, br.nblk, static_cast<int>(per_field)));
  ctx->launches += 2;
  WB2_TRY(pk.release());
  return WB2_OK;
}

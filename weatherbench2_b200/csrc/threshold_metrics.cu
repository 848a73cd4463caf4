// K7 -- threshold ("binary event") and Gaussian-forecast metrics (sm_90a).
//
// Ensemble entry (wb2_ens_threshold_metrics): EnsembleBrierScore /
// DebiasedEnsembleBrierScore (weatherbench2/metrics.py:1523-1710),
// EnsembleIgnoranceScore (:1713-1790), EnsembleRPS (:1793-1891).  One read of
// the M members yields, for every threshold of the pass, the counts
// #{x_m > thr}, #{x_m < thr}, #{x_m not NaN}; the four point-wise scores follow
// from the counts and are reduced with the same weight machinery as K1 / K2.
//
// Gaussian entry (wb2_gaussian_metrics): GaussianCRPS / GaussianVariance
// (:849-937) and GaussianBrierScore / IgnoranceScore / RPS (:963-1158) from a
// (mean, std) forecast.  The reference evaluates scipy.stats.norm in float64;
// here z = (thr - mean) / std is rounded to float32 and erfcf / expf / logf /
// log1pf run in float32 on min(cdf, 1 - cdf), which they keep to a few ulp
// relative.  Past tail < 1e-7 (|z| > 5.2) the tail is recomputed with float64
// erfc from the float32 z and the reference's float64 `1 - cdf` is replayed,
// so the ignorance saturates to inf where the reference's does (tail <= 2^-54).
//
// Thresholds are either read from a float32 field per (threshold, field)
// (QuantileThreshold, thresholds.py:118-149) or built in the kernel from the
// climatological mean and std, thr = mean + z_q * std in float64
// (GaussianQuantileThreshold, thresholds.py:152-185) -- the same two roundings
// as the reference -- and compared exactly: for a float32 x,
//   x > thr  <=>  x > round_down_f32(thr),   x < thr  <=>  x < round_up_f32(thr).
#include <cmath>

#include "region_reduce.cuh"

namespace wb2 {

constexpr int kThrWarps = 4;
constexpr int kThrThreads = kThrWarps * 32;
constexpr int kThrStats = 4;            // brier, debiased brier, ignorance, rps part
constexpr int kThrOut = 2 * kThrStats;  // + the four weight sums

struct ThrParams {
  const float* x;  // ensemble (member 0) or Gaussian mean forecast
  const float* s;  // Gaussian forecast std (Gaussian entry only)
  const float* t;
  const float* thr_a;  // thresholds, or climatological mean (Gaussian-quantile mode)
  const float* thr_b;  // climatological std (Gaussian-quantile mode) or null
  const int64_t* off_x;
  const int64_t* off_s;
  const int64_t* off_t;
  const int64_t* off_a;  // field thresholds: [nq][nfield]; Gaussian-quantile: [nfield]
  const int64_t* off_b;  // [nfield]
  const double* z;       // [nq] standard-normal quantiles (Gaussian-quantile mode)
  const double* row_w;
  const int32_t* seg_start;
  const double* seg_w;
  const float* col_w;
  const float* cell_w;
  double* partial;  // [nfield][nblk][nq][R][kThrOut]
  int64_t member_stride, row_stride, nfield;
  int32_t nmember, nrow, ncol, nregion, nseg, zero_skip, rows_per_block, nblk, nq, q0;
};

// thresholds of one grid point for the TQ thresholds of this pass: the float64
// threshold and the float32 bracket [lo, hi] used for exact comparisons
template <int TQ>
__device__ __forceinline__ void load_thresholds(const ThrParams& p, int64_t field, int64_t cell,
                                                float (&lo)[TQ], float (&hi)[TQ],
                                                double (&thr)[TQ]) {
  if (p.thr_b != nullptr) {
    const double mean = double(ldg_stream(p.thr_a + p.off_a[field] + cell));
    const double sd = double(ldg_stream(p.thr_b + p.off_b[field] + cell));
#pragma unroll
    for (int q = 0; q < TQ; ++q) {
      // thresholds.py:182-184: mean + ppf(q) * std, two float64 roundings
      thr[q] = p.q0 + q < p.nq ? __dadd_rn(mean, __dmul_rn(p.z[p.q0 + q], sd)) : 0.0;
      lo[q] = __double2float_rd(thr[q]);
      hi[q] = __double2float_ru(thr[q]);
    }
  } else {
#pragma unroll
    for (int q = 0; q < TQ; ++q) {
      float v = 0.f;
      if (p.q0 + q < p.nq)
        v = ldg_stream(p.thr_a + p.off_a[int64_t(p.q0 + q) * p.nfield + field] + cell);
      lo[q] = hi[q] = v;
      thr[q] = double(v);
    }
  }
}

// weighted accumulation shared by both kernels: per-lane float partials of one
// (row, segment) -> warp butterfly -> lane r applies region r's float64 weight.
template <int NV, bool SKIPNA>
struct SegAcc {
  float sum[NV];
  float wsum[SKIPNA ? NV : 1];
  __device__ __forceinline__ void clear() {
#pragma unroll
    for (int i = 0; i < NV; ++i) sum[i] = 0.f;
#pragma unroll
    for (int i = 0; i < (SKIPNA ? NV : 1); ++i) wsum[i] = 0.f;
  }
  __device__ __forceinline__ void add(const float (&val)[NV], float wc) {
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      if (SKIPNA) {
        if (val[i] == val[i]) { sum[i] += wc * val[i]; wsum[i] += wc; }
      } else {
        sum[i] += wc * val[i];
      }
    }
    if (!SKIPNA) wsum[0] += wc;
  }
};

// Point-wise ensemble scores for the TQ thresholds of a pass: counts over the
// streamed members, then Brier / debiased Brier / ignorance / RPS part.
// c / d given inv ~= 1 / d: one Newton step on the quotient (three
// instructions; exact quotients such as M / M = 1 come out exact, which the
// known-answer tests with expected 0 rely on).
__device__ __forceinline__ float div_by(float c, float d, float inv) {
  const float q = c * inv;
  return fmaf(fmaf(-d, q, c), inv, q);
}

template <int TQ, bool SKIPNA>
__device__ __forceinline__ void ens_threshold_point(const float* __restrict__ src,
                                                    int64_t member_stride, int M, float t,
                                                    const float (&lo)[TQ], const float (&hi)[TQ],
                                                    int nq_left, float (&val)[TQ * kThrStats]) {
  const float nanv = __int_as_float(0x7fc00000);
  // ---- ensemble: counts over the members ----------------------------------
  float c_gt[TQ], c_lt[TQ];
#pragma unroll
  for (int q = 0; q < TQ; ++q) { c_gt[q] = 0.f; c_lt[q] = 0.f; }
  float nvalid = 0.f;
    // A float64 threshold that is not a float32 number has lo < hi
  // (adjacent floats), and then  #{x < hi} = #valid - #{x > lo}: one
  // comparison per (member, threshold) instead of two.
  bool strict = true;
#pragma unroll
  for (int q = 0; q < TQ; ++q) strict = strict && (lo[q] < hi[q] || q >= nq_left);
  if (__all_sync(__activemask(), strict)) {
#pragma unroll 25
    for (int m = 0; m < M; ++m) {
      const float xm = ldg_stream(src + int64_t(m) * member_stride);
      nvalid += (xm == xm) ? 1.f : 0.f;
#pragma unroll
      for (int q = 0; q < TQ; ++q) c_gt[q] += (xm > lo[q]) ? 1.f : 0.f;
    }
#pragma unroll
    for (int q = 0; q < TQ; ++q) c_lt[q] = nvalid - c_gt[q];
  } else {
#pragma unroll 25
    for (int m = 0; m < M; ++m) {
      const float xm = ldg_stream(src + int64_t(m) * member_stride);
      nvalid += (xm == xm) ? 1.f : 0.f;
#pragma unroll
      for (int q = 0; q < TQ; ++q) {
        c_gt[q] += (xm > lo[q]) ? 1.f : 0.f;
        c_lt[q] += (xm < hi[q]) ? 1.f : 0.f;
      }
    }
  }
  const float fm = float(M);
  const bool t_nan = !(t == t);
  // every division below is by M, the valid count or one less: three
  // reciprocals per point instead of five IEEE divisions per threshold (a
  // ~15-instruction subroutine each: ~40 % of this function's instructions at
  // four thresholds); <= 1 ulp apart, 0 * inf keeps the 0 / 0 -> NaN cases
  const float inv_fm = 1.f / fm;
  const float nv = SKIPNA ? nvalid : fm;
  const float inv_nv = SKIPNA ? 1.f / nv : inv_fm;
  const float inv_nv1 = 1.f / (nv - 1.f);
#pragma unroll
  for (int q = 0; q < TQ; ++q) {
    // Brier (metrics.py:1523-1560): NaN-aware probabilities
    float pf = div_by(c_gt[q], nv, inv_nv);  // 0 / 0 -> NaN like nanmean of nothing
    if (!SKIPNA && nvalid < fm) pf = nanv;
    const float tp = t_nan ? nanv : (t > lo[q] ? 1.f : 0.f);
    const float d = pf - tp;
    const float brier = d * d;
    // ddof = 1 variance of the 0 / 1 member probabilities (:545-565)
    const float q1 = 1.f - pf;
    float var = (c_gt[q] * q1 * q1 + (nv - c_gt[q]) * pf * pf) * inv_nv1;
    if (SKIPNA && !(nvalid > 1.f)) var = nanv;
    // ignorance (:1713-1729) and RPS part (:1793-1803): plain 0 / 1
    // indicators, a NaN member counts as "not above" / "not below"
    const bool t_gt = t > lo[q];
    const float pi = div_by(t_gt ? c_gt[q] : fm - c_gt[q], fm, inv_fm);
    const float dr = div_by(c_lt[q], fm, inv_fm) - (t < hi[q] ? 1.f : 0.f);
    val[q * kThrStats + 0] = brier;
    val[q * kThrStats + 1] = brier - var * inv_fm;
    val[q * kThrStats + 2] = -logf(pi);
    val[q * kThrStats + 3] = dr * dr;
  }
}

template <int TQ, bool SKIPNA, bool GAUSS>
__global__ void __launch_bounds__(kThrThreads, 4) threshold_kernel(const ThrParams p) {
  constexpr int NV = TQ * kThrStats;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double* red = reinterpret_cast<double*>(smem_raw);  // [warps][32][2 * NV]
  float* s_colw = reinterpret_cast<float*>(red + kThrWarps * 32 * 2 * NV);

  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int64_t field = blockIdx.x / p.nblk;
  const int blk = blockIdx.x % p.nblk;
  const int R = p.nregion;
  const int M = p.nmember;
  const bool weighted = p.col_w != nullptr || p.cell_w != nullptr;
  if (p.col_w) {
    for (int i = threadIdx.x; i < p.ncol; i += kThrThreads) s_colw[i] = p.col_w[i];
    __syncthreads();
  }
  const float* __restrict__ px = p.x + p.off_x[field];
  const float* __restrict__ ps = GAUSS ? p.s + p.off_s[field] : nullptr;
  const float* __restrict__ pt = p.t + p.off_t[field];
  const bool zero_skip = p.zero_skip != 0;
  const float nanv = __int_as_float(0x7fc00000);

  // float64 accumulators live in shared memory (touched once per row segment):
  // keeping 2 * NV doubles in registers would cost occupancy, and this kernel
  // needs many member loads in flight.
  double* accd = red + (warp * 32 + lane) * 2 * NV;
#pragma unroll
  for (int i = 0; i < 2 * NV; ++i) accd[i] = 0.0;

  const int row0 = blk * p.rows_per_block;
  const int row1 = min(p.nrow, row0 + p.rows_per_block);
  for (int row = row0 + warp; row < row1; row += kThrWarps) {
    const int64_t rbase = int64_t(row) * p.row_stride;
    for (int k = 0; k < p.nseg; ++k) {
      const int cs = p.seg_start[k];
      const int ce = p.seg_start[k + 1];
      SegAcc<NV, SKIPNA> acc;
      acc.clear();
      // Gaussian entry: a cell is three loads followed by ~130 dependent
      // instructions (erfc, exp, log); ncu showed 12.5 warps per issue waiting on
      // the long scoreboard of those loads.  The operands of the next two
      // cells of this lane are therefore fetched ahead (a 2-deep register ring:
      // 0.17 -> 0.26 of the HBM roofline; four cells ahead cost occupancy: 0.22).
      constexpr int PD = 2;  // prefetch depth (cells of this lane ahead)
      float pf_t[PD], pf_m[PD], pf_s[PD];
#pragma unroll
      for (int j = 0; j < PD; ++j) { pf_t[j] = 0.f; pf_m[j] = 0.f; pf_s[j] = 1.f; }
      if (GAUSS) {
#pragma unroll
        for (int j = 0; j < PD; ++j) {
          const int c2 = cs + lane + 32 * j;
          if (c2 < ce) {
            pf_t[j] = ldg_stream(pt + rbase + c2);
            pf_m[j] = ldg_stream(px + rbase + c2);
            pf_s[j] = ldg_stream(ps + rbase + c2);
          }
        }
      }
      for (int col = cs + lane; col < ce; col += 32) {
        float g_t = 0.f, g_m = 0.f, g_s = 1.f;
        if (GAUSS) {  // rotate the prefetch ring and refill its tail
          g_t = pf_t[0]; g_m = pf_m[0]; g_s = pf_s[0];
#pragma unroll
          for (int j = 0; j + 1 < PD; ++j) {
            pf_t[j] = pf_t[j + 1]; pf_m[j] = pf_m[j + 1]; pf_s[j] = pf_s[j + 1];
          }
          const int c2 = col + 32 * PD;
          if (c2 < ce) {
            pf_t[PD - 1] = ldg_stream(pt + rbase + c2);
            pf_m[PD - 1] = ldg_stream(px + rbase + c2);
            pf_s[PD - 1] = ldg_stream(ps + rbase + c2);
          }
        }
        float wc = 1.f;
        if (weighted) {
          if (p.col_w) wc *= s_colw[col];
          if (p.cell_w) wc *= p.cell_w[int64_t(row) * p.ncol + col];
          if (zero_skip && wc == 0.f) continue;  // metrics.py:160
        }
        const int64_t cell = rbase + col;
        const float t = GAUSS ? g_t : ldg_stream(pt + cell);
        float lo[TQ], hi[TQ];
        double thr[TQ];
        load_thresholds<TQ>(p, field, cell, lo, hi, thr);
        float val[NV];
        if (GAUSS) {
          // ---- Gaussian forecast N(mean, std) ----------------------------------
          // The reference evaluates scipy.stats.norm in float64.  erfc / exp in
          // float64 would make this kernel FP64-bound (measured 0.02-0.09 of
          // the HBM roofline), so the transcendental part runs in float32 --
          // always on the tail where erfcf keeps full RELATIVE accuracy -- and
          // only the far tail (below 1e-7, rare) goes back to float64, where
          // the reference's `1 - cdf` rounding step is replayed (it decides
          // when the ignorance score saturates to inf).
          const float mean = g_m;
          const float sd = g_s;
          if (p.nq == 0) {
            // GaussianCRPS (metrics.py:889-899) and GaussianVariance (:918-922)
            const float zn = (mean - t) / sd;
            const float az = fabsf(zn);
            // |z| (2 Phi(|z|) - 1) = |z| (1 - erfc(|z| / sqrt 2)): even in z
            const float tail = erfcf(az * 0.70710678f);
            const float pdf = 0.39894228f * expf(-0.5f * zn * zn);
            val[0] = sd * (az * (1.f - tail) + 2.f * pdf - 0.56418958f);
            val[1] = sd * sd;
#pragma unroll
            for (int i = 2; i < NV; ++i) val[i] = 0.f;
          } else {
            const float rsd = 1.f / sd;  // one division per cell, not per threshold
#pragma unroll
            for (int q = 0; q < TQ; ++q) {
              // metrics.py:972, 1040, 1112
              const float zn = float(thr[q] - double(mean)) * rsd;
              const float tail = 0.5f * erfcf(fabsf(zn) * 0.70710678f);  // min(cdf, 1 - cdf)
              const bool up = zn > 0.f;     // cdf = up ? 1 - tail : tail
              const bool t_gt = t > lo[q];  // truth > threshold (NaN -> false)
              const bool t_lt = t < hi[q];
              float brier, ign, rps;
              if (tail >= 1e-7f) {
                // float32 is enough away from the far tail: each score needs
                // either `tail` itself (full relative accuracy) or 1 - tail
                // (absolute accuracy 6e-8), never their difference:
                //   pe - [t > thr]  = t_gt ? -cdf : pe,   cdf - [t < thr] = t_lt ? -pe : cdf
                const float one_m = 1.f - tail;
                const float cdf = up ? one_m : tail, pe = up ? tail : one_m;
                const float db = t_gt ? cdf : pe, dr = t_lt ? pe : cdf;
                brier = db * db;
                rps = dr * dr;
                // -log(t_gt ? pe : cdf): the argument is `tail` iff t_gt == up
                ign = (t_gt == up) ? -logf(tail) : -log1pf(-tail);
              } else {
                // far tail (|z| > 5.2): the tail again in float64 -- erfcf
                // goes subnormal at |z| ~ 13 and to 0 at |z| ~ 14, where the
                // reference's float64 cdf is finite down to |z| ~ 38 -- and
                // the reference's float64 `1 - cdf` rounding replayed on it:
                // it decides where the ignorance saturates to inf.  scipy's
                // erfc returns 0 once a^2 > 709.78 (|z| > 37.68) where CUDA's
                // returns a subnormal; the reference's cdf is 0 there.
                const double a = double(fabsf(zn)) * 0.70710678118654752;
                const double tl = a * a > 709.782712893384 ? 0.0 : 0.5 * erfc(a);
                const double cdf = up ? 1.0 - tl : tl;
                const double pe = 1.0 - cdf;  // exceedance probability
                const double db = pe - (t_gt ? 1.0 : 0.0);
                const double dr = cdf - (t_lt ? 1.0 : 0.0);
                brier = float(db * db);
                rps = float(dr * dr);
                ign = float(-log(t_gt ? pe : cdf));
              }
              val[q * kThrStats + 0] = brier;  // :980
              val[q * kThrStats + 1] = 0.f;
              val[q * kThrStats + 2] = ign;    // :1044-1048
              val[q * kThrStats + 3] = rps;    // :1118
            }
          }
        } else {
          ens_threshold_point<TQ, SKIPNA>(px + cell, p.member_stride, M, t, lo, hi, p.nq - p.q0,
                                          val);
        }
        acc.add(val, wc);
      }
#pragma unroll
      for (int i = 0; i < NV; ++i) acc.sum[i] = warp_sum(acc.sum[i]);
#pragma unroll
      for (int i = 0; i < (SKIPNA ? NV : 1); ++i) acc.wsum[i] = warp_sum(acc.wsum[i]);
      if (lane < R) {
        const double w = p.row_w[int64_t(lane) * p.nrow + row] * p.seg_w[lane * p.nseg + k];
        if (!(zero_skip && w == 0.0)) {
#pragma unroll
          for (int i = 0; i < NV; ++i) {
            accd[i] += w * double(acc.sum[i]);
            accd[NV + i] += w * double(acc.wsum[SKIPNA ? i : 0]);
          }
        }
      }
    }
  }

  __syncthreads();
  // partial layout: [field][blk][q][r][sums(4), weight sums(4)]
  double* out = p.partial + (field * p.nblk + blk) * int64_t(p.nq > 0 ? p.nq : 1) * R * kThrOut;
  const int nq_here = p.nq > 0 ? min(TQ, p.nq - p.q0) : 1;
  for (int idx = threadIdx.x; idx < nq_here * R * kThrOut; idx += kThrThreads) {
    const int q = idx / (R * kThrOut);
    const int r = (idx / kThrOut) % R;
    const int st = idx % kThrOut;
    const int slot = st < kThrStats ? q * kThrStats + st : NV + q * kThrStats + (st - kThrStats);
    double v = 0.0;
#pragma unroll
    for (int w = 0; w < kThrWarps; ++w) v += red[(w * 32 + r) * 2 * NV + slot];
    out[(int64_t(p.q0 + q) * R + r) * kThrOut + st] = v;
  }
}

template <int TQ, bool GAUSS>
static int launch_threshold(wb2_ctx* ctx, const ThrParams& p, int64_t nfield, bool skipna) {
  const size_t smem = size_t(kThrWarps) * 32 * 2 * TQ * kThrStats * sizeof(double) +
                      (p.col_w ? size_t(p.ncol) * sizeof(float) : 0);
  const dim3 grid(static_cast<unsigned>(nfield * p.nblk));
  auto go = [&](auto kernel) { return launch_kernel(ctx, kernel, grid, kThrThreads, smem, p); };
  return skipna ? go(threshold_kernel<TQ, true, GAUSS>) : go(threshold_kernel<TQ, false, GAUSS>);
}

// Shared host driver of the two entry points.
static int threshold_impl(wb2_ctx* ctx, bool gauss, const float* x, const float* s, const float* t,
                          const float* thr_a, const float* thr_b, const double* z, int32_t nq,
                          int32_t nmember, int64_t member_stride, int64_t nfield,
                          const int64_t* off_x, const int64_t* off_s, const int64_t* off_t,
                          const int64_t* off_a, const int64_t* off_b, const wb2_weights* w,
                          int skipna, double* out) {
  const BlockRows br = block_rows(w->nrow, nfield, 2 * kThrWarps, kThrWarps, 4 * ctx->num_sms);
  const int nq_out = nq > 0 ? nq : 1;
  const size_t per_field = size_t(nq_out) * w->nregion * kThrOut;
  const bool gq = thr_b != nullptr;
  Packer pk(ctx);
  const size_t o_x = pk.add(off_x, nfield * sizeof(int64_t));
  const size_t o_s = gauss ? pk.add(off_s, nfield * sizeof(int64_t)) : 0;
  const size_t o_t = pk.add(off_t, nfield * sizeof(int64_t));
  const size_t o_a = nq > 0 ? pk.add(off_a, size_t(gq ? 1 : nq) * nfield * sizeof(int64_t)) : 0;
  const size_t o_b = gq ? pk.add(off_b, nfield * sizeof(int64_t)) : 0;
  const size_t o_z = gq ? pk.add(z, size_t(nq) * sizeof(double)) : 0;
  const WeightUpload wu(pk, w);
  const size_t o_part = pk.reserve(size_t(nfield) * br.nblk * per_field * sizeof(double));
  WB2_TRY(pk.commit());

  ThrParams p;
  p.x = x; p.s = s; p.t = t; p.thr_a = thr_a; p.thr_b = thr_b;
  p.off_x = pk.dev<int64_t>(o_x);
  p.off_s = gauss ? pk.dev<int64_t>(o_s) : nullptr;
  p.off_t = pk.dev<int64_t>(o_t);
  p.off_a = nq > 0 ? pk.dev<int64_t>(o_a) : nullptr;
  p.off_b = gq ? pk.dev<int64_t>(o_b) : nullptr;
  p.z = gq ? pk.dev<double>(o_z) : nullptr;
  wu.bind(p);
  p.partial = pk.dev<double>(o_part);
  p.member_stride = member_stride;
  p.nfield = nfield;
  p.nmember = nmember;
  p.rows_per_block = br.rows_per_block; p.nblk = br.nblk;
  p.nq = nq;
  const bool sk = skipna != 0;
  int launches = 0;
  for (int q0 = 0; q0 < nq_out;) {
    const int left = nq_out - q0;
    p.q0 = q0;
    int rc;
    if (gauss) {
      if (left >= 4) { rc = launch_threshold<4, true>(ctx, p, nfield, sk); q0 += 4; }
      else if (left >= 2) { rc = launch_threshold<2, true>(ctx, p, nfield, sk); q0 += 2; }
      else { rc = launch_threshold<1, true>(ctx, p, nfield, sk); q0 += 1; }
    } else {
      if (left >= 4) { rc = launch_threshold<4, false>(ctx, p, nfield, sk); q0 += 4; }
      else if (left >= 2) { rc = launch_threshold<2, false>(ctx, p, nfield, sk); q0 += 2; }
      else { rc = launch_threshold<1, false>(ctx, p, nfield, sk); q0 += 1; }
    }
    if (rc != WB2_OK) return rc;
    ++launches;
  }
  WB2_TRY(launch_block_sum(ctx, p.partial, out, nfield, br.nblk, static_cast<int>(per_field)));
  ctx->launches += launches + 1;
  WB2_TRY(pk.release());
  return WB2_OK;
}

static int check_threshold_args(const wb2_ctx* ctx, int dtype, int32_t nq, const void* thr_a,
                                const void* thr_b, const int64_t* off_a, const int64_t* off_b,
                                const double* z, const wb2_weights* w, const double* out,
                                int64_t nfield) {
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_REQUIRE(dtype == WB2_F32, "threshold metrics: only WB2_F32 inputs are supported");
  WB2_REQUIRE(nq >= 0 && nq <= 4096, "nthreshold out of range");
  WB2_TRY(validate_weights(w));
  WB2_REQUIRE(out != nullptr, "out is NULL");
  WB2_REQUIRE(nfield >= 0 && nfield <= (int64_t(1) << 24), "nfield out of range");
  if (nq > 0) {
    WB2_REQUIRE(thr_a && off_a, "thresholds and their offset table must not be NULL");
    if (thr_b) WB2_REQUIRE(off_b && z, "Gaussian-quantile thresholds need off_b and z");
  }
  return WB2_OK;
}

}  // namespace wb2

using namespace wb2;

extern "C" int wb2_ens_threshold_metrics(wb2_ctx* ctx, const void* x, const void* t, int dtype,
                                         int32_t nmember, int64_t member_stride, int64_t nfield,
                                         const int64_t* off_x, const int64_t* off_t,
                                         int32_t nthreshold, const void* thr_a,
                                         const int64_t* off_a, const void* thr_b,
                                         const int64_t* off_b, const double* z,
                                         const wb2_weights* w, int skipna, double* out) {
  WB2_NVTX("wb2_ens_threshold_metrics");
  WB2_TRY(check_threshold_args(ctx, dtype, nthreshold, thr_a, thr_b, off_a, off_b, z, w, out,
                               nfield));
  WB2_REQUIRE(nthreshold >= 1, "wb2_ens_threshold_metrics: nthreshold must be >= 1");
  WB2_REQUIRE(nmember >= 1 && nmember <= 65536, "nmember out of range");
  if (nfield == 0) return WB2_OK;
  WB2_REQUIRE(x && t && off_x && off_t, "x/t and their offset tables must not be NULL");
  DeviceGuard guard(ctx->device);
  return threshold_impl(ctx, false, static_cast<const float*>(x), nullptr,
                        static_cast<const float*>(t), static_cast<const float*>(thr_a),
                        static_cast<const float*>(thr_b), z, nthreshold, nmember, member_stride,
                        nfield, off_x, nullptr, off_t, off_a, off_b, w, skipna, out);
}

extern "C" int wb2_gaussian_metrics(wb2_ctx* ctx, const void* mean, const void* std,
                                    const void* t, int dtype, int64_t nfield,
                                    const int64_t* off_mean, const int64_t* off_std,
                                    const int64_t* off_t, int32_t nthreshold, const void* thr_a,
                                    const int64_t* off_a, const void* thr_b,
                                    const int64_t* off_b, const double* z, const wb2_weights* w,
                                    int skipna, double* out) {
  WB2_NVTX("wb2_gaussian_metrics");
  WB2_TRY(check_threshold_args(ctx, dtype, nthreshold, thr_a, thr_b, off_a, off_b, z, w, out,
                               nfield));
  if (nfield == 0) return WB2_OK;
  WB2_REQUIRE(mean && std && t && off_mean && off_std && off_t,
              "mean/std/t and their offset tables must not be NULL");
  DeviceGuard guard(ctx->device);
  return threshold_impl(ctx, true, static_cast<const float*>(mean),
                        static_cast<const float*>(std), static_cast<const float*>(t),
                        static_cast<const float*>(thr_a), static_cast<const float*>(thr_b), z,
                        nthreshold, 1, 0, nfield, off_mean, off_std, off_t, off_a, off_b, w,
                        skipna, out);
}

// ---- map output (SpatialEnsembleBrierScore & co.) -------------------------------
// One thread per grid cell of one output map; walks the ngroup (time) slabs that
// average into it, like K6e.  One statistic per launch, TQ thresholds per pass.
namespace wb2 {

struct ThrMapExtra {
  float* out;  // [nq][nout][nrow][ncol]
  int64_t nout, cells_per_map;
  int32_t ngroup, stat, bpm;
};

template <int TQ, bool SKIPNA>
__global__ void __launch_bounds__(kThrThreads, 4)
    threshold_maps_kernel(const ThrParams p, const ThrMapExtra e) {
  const int64_t j = blockIdx.x / e.bpm;
  const int64_t ci = int64_t(blockIdx.x % e.bpm) * kThrThreads + threadIdx.x;
  if (ci >= e.cells_per_map) return;
  const int row = static_cast<int>(ci / p.ncol);
  const int col = static_cast<int>(ci % p.ncol);
  const int64_t cell = int64_t(row) * p.row_stride + col;
  double acc[TQ];
  int cnt[TQ];
  float last[TQ];
#pragma unroll
  for (int q = 0; q < TQ; ++q) { acc[q] = 0.0; cnt[q] = 0; last[q] = 0.f; }
  for (int g = 0; g < e.ngroup; ++g) {
    const int64_t field = j * e.ngroup + g;
    const float t = ldg_stream(p.t + p.off_t[field] + cell);
    float lo[TQ], hi[TQ];
    double thr[TQ];
    load_thresholds<TQ>(p, field, cell, lo, hi, thr);
    float val[TQ * kThrStats];
    ens_threshold_point<TQ, SKIPNA>(p.x + p.off_x[field] + cell, p.member_stride, p.nmember, t, lo,
                                    hi, p.nq - p.q0, val);
#pragma unroll
    for (int q = 0; q < TQ; ++q) {
      const float* vq = val + q * kThrStats;
      const float v = e.stat == 0 ? vq[0] : (e.stat == 1 ? vq[1] : (e.stat == 2 ? vq[2] : vq[3]));
      last[q] = v;
      if (SKIPNA) {
        if (v == v) { acc[q] += double(v); ++cnt[q]; }
      } else {
        acc[q] += double(v);
      }
    }
  }
#pragma unroll
  for (int q = 0; q < TQ; ++q) {
    if (p.q0 + q >= p.nq) continue;
    float r;
    if (e.ngroup == 1) r = last[q];
    else if (SKIPNA) r = cnt[q] > 0 ? float(acc[q] / double(cnt[q])) : __int_as_float(0x7fc00000);
    else r = float(acc[q] / double(e.ngroup));
    e.out[(int64_t(p.q0 + q) * e.nout + j) * e.cells_per_map + ci] = r;
  }
}

template <int TQ>
static int launch_threshold_maps(wb2_ctx* ctx, const ThrParams& p, const ThrMapExtra& e,
                                 bool skipna) {
  const dim3 grid(static_cast<unsigned>(e.nout * e.bpm));
  if (skipna) threshold_maps_kernel<TQ, true><<<grid, kThrThreads, 0, ctx->stream>>>(p, e);
  else threshold_maps_kernel<TQ, false><<<grid, kThrThreads, 0, ctx->stream>>>(p, e);
  WB2_CUDA_TRY(cudaGetLastError());
  return WB2_OK;
}

}  // namespace wb2

extern "C" int wb2_ens_threshold_maps(wb2_ctx* ctx, const void* x, const void* t, int dtype,
                                      int32_t nmember, int64_t member_stride, int64_t nout,
                                      int32_t ngroup, const int64_t* off_x, const int64_t* off_t,
                                      int32_t nthreshold, const void* thr_a, const int64_t* off_a,
                                      const void* thr_b, const int64_t* off_b, const double* z,
                                      int32_t nrow, int32_t ncol, int64_t row_stride, int32_t stat,
                                      int skipna, float* out) {
  WB2_NVTX("wb2_ens_threshold_maps");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_REQUIRE(dtype == WB2_F32, "wb2_ens_threshold_maps: only WB2_F32 inputs are supported");
  WB2_REQUIRE(nthreshold >= 1 && nthreshold <= 4096, "nthreshold out of range");
  WB2_REQUIRE(nmember >= 1 && nmember <= 65536, "nmember out of range");
  WB2_REQUIRE(stat >= 0 && stat < kThrStats, "stat must be 0..3 (brier, debiased, ignorance, rps)");
  WB2_REQUIRE(nrow > 0 && ncol > 0 && row_stride >= ncol, "bad grid: nrow=%d ncol=%d", nrow, ncol);
  WB2_REQUIRE(nout >= 0 && ngroup >= 1, "nout must be >= 0 and ngroup >= 1");
  if (nout == 0) return WB2_OK;
  WB2_REQUIRE(x && t && off_x && off_t && out && thr_a && off_a,
              "x/t/out/thresholds and their offset tables must not be NULL");
  if (thr_b) WB2_REQUIRE(off_b && z, "Gaussian-quantile thresholds need off_b and z");
  DeviceGuard guard(ctx->device);
  const int64_t nfield = nout * ngroup;
  const bool gq = thr_b != nullptr;
  Packer pk(ctx);
  const size_t o_x = pk.add(off_x, nfield * sizeof(int64_t));
  const size_t o_t = pk.add(off_t, nfield * sizeof(int64_t));
  const size_t o_a = pk.add(off_a, size_t(gq ? 1 : nthreshold) * nfield * sizeof(int64_t));
  const size_t o_b = gq ? pk.add(off_b, nfield * sizeof(int64_t)) : 0;
  const size_t o_z = gq ? pk.add(z, size_t(nthreshold) * sizeof(double)) : 0;
  WB2_TRY(pk.commit());
  ThrParams p = {};
  p.x = static_cast<const float*>(x);
  p.t = static_cast<const float*>(t);
  p.thr_a = static_cast<const float*>(thr_a);
  p.thr_b = static_cast<const float*>(thr_b);
  p.off_x = pk.dev<int64_t>(o_x);
  p.off_t = pk.dev<int64_t>(o_t);
  p.off_a = pk.dev<int64_t>(o_a);
  p.off_b = gq ? pk.dev<int64_t>(o_b) : nullptr;
  p.z = gq ? pk.dev<double>(o_z) : nullptr;
  p.member_stride = member_stride;
  p.row_stride = row_stride;
  p.nfield = nfield;
  p.nmember = nmember;
  p.nrow = nrow; p.ncol = ncol;
  p.nq = nthreshold;
  ThrMapExtra e;
  e.out = out;
  e.nout = nout;
  e.cells_per_map = int64_t(nrow) * ncol;
  e.ngroup = ngroup;
  e.stat = stat;
  e.bpm = static_cast<int32_t>((e.cells_per_map + kThrThreads - 1) / kThrThreads);
  WB2_REQUIRE(nout * int64_t(e.bpm) < (int64_t(1) << 31), "launch too large");
  int launches = 0;
  for (int q0 = 0; q0 < nthreshold;) {
    const int left = nthreshold - q0;
    p.q0 = q0;
    int rc;
    if (left >= 4) { rc = launch_threshold_maps<4>(ctx, p, e, skipna != 0); q0 += 4; }
    else if (left >= 2) { rc = launch_threshold_maps<2>(ctx, p, e, skipna != 0); q0 += 2; }
    else { rc = launch_threshold_maps<1>(ctx, p, e, skipna != 0); q0 += 1; }
    if (rc != WB2_OK) return rc;
    ++launches;
  }
  ctx->launches += launches;
  WB2_TRY(pk.release());
  return WB2_OK;
}

// Point-wise ensemble statistics shared by K2 (ens_metrics.cu, spatially
// averaged) and K6e (ens_maps.cu, map output): the M members of one grid point
// sit in registers and pass through a Batcher sorting network.
#pragma once
#include "common.cuh"

namespace wb2 {

// Two float32 in one 64-bit register pair (lane 0 = lo, lane 1 = hi).  sm_90
// has no packed FP32 instruction, so every pair operation is two scalar IEEE
// round-to-nearest operations (the __f*_rn intrinsics are never contracted):
// each lane rounds exactly as a packed .f32x2 operation would.
typedef unsigned long long u64x2f;

__device__ __forceinline__ u64x2f pk2f(float lo, float hi) {
  u64x2f r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
  return r;
}
__device__ __forceinline__ void unpk2f(u64x2f v, float& lo, float& hi) {
  asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
__device__ __forceinline__ u64x2f add2f(u64x2f a, u64x2f b) {
  float a0, a1, b0, b1;
  unpk2f(a, a0, a1);
  unpk2f(b, b0, b1);
  return pk2f(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
__device__ __forceinline__ u64x2f sub2f(u64x2f a, u64x2f b) {
  float a0, a1, b0, b1;
  unpk2f(a, a0, a1);
  unpk2f(b, b0, b1);
  return pk2f(__fsub_rn(a0, b0), __fsub_rn(a1, b1));
}
__device__ __forceinline__ u64x2f fma2f(u64x2f a, u64x2f b, u64x2f c) {
  float a0, a1, b0, b1, c0, c1;
  unpk2f(a, a0, a1);
  unpk2f(b, b0, b1);
  unpk2f(c, c0, c1);
  return pk2f(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}

// compare-exchange of one element (scalar members of one grid point)
__device__ __forceinline__ void ce_any(float& a, float& b) {
  const float lo_ = fminf(a, b);
  const float hi_ = fmaxf(a, b);
  a = lo_;
  b = hi_;
}
// compare-exchange of the SAME comparator on two adjacent grid points held as
// one pair per member (ens_pair_kernel): the two minima are FMNMX (ALU pipe),
// the two maxima come from hi = (a + b) - lo as FADDs (FMA pipe) -- the
// comparators are split between the two pipes, and the pairs need no register
// shuffling because they are loaded as pairs (LDG.64).  Inexact by one
// rounding of the pair sum: only used on mean-removed members.
__device__ __forceinline__ void ce_any(u64x2f& a, u64x2f& b) {
  float a0, a1, b0, b1;
  unpk2f(a, a0, a1);
  unpk2f(b, b0, b1);
  const u64x2f lo = pk2f(fminf(a0, b0), fminf(a1, b1));
  b = sub2f(add2f(a, b), lo);
  a = lo;
}
// exact variant of the pair comparator: maxima on the ALU pipe too
__device__ __forceinline__ void ce_any_minmax(u64x2f& a, u64x2f& b) {
  float a0, a1, b0, b1;
  unpk2f(a, a0, a1);
  unpk2f(b, b0, b1);
  a = pk2f(fminf(a0, b0), fminf(a1, b1));
  b = pk2f(fmaxf(a0, b0), fmaxf(a1, b1));
}
// Comparator K of the generated networks.  Scalar members: always min / max.
// Pairs: two of three comparators take the (a + b) - lo form, every third one
// min / max, which splits the work between the FMA pipe (that also does the
// moment sums) and the ALU pipe.
template <int K>
__device__ __forceinline__ void ce_sel(float& a, float& b) { ce_any(a, b); }
template <int K>
__device__ __forceinline__ void ce_sel(u64x2f& a, u64x2f& b) {
  if (K % 3 == 0) ce_any_minmax(a, b);
  else ce_any(a, b);
}
#define CE(a, b) ce_sel<__COUNTER__>(v[a], v[b]);
// Twin compare-exchange on two aligned register pairs (v[a], v[a+1]) and
// (v[b], v[b+1]): the minima cost one FMNMX each (ALU pipe, one warp
// instruction per 2 cycles per SM sub-partition), the maxima come from
// hi = (a + b) - lo as FADDs on the FMA pipe, which moves half of those
// comparators' work off the ALU pipe.  (a + b) - lo is not exact: it is only
// used on mean-removed members, where the rounding error is relative to the
// ensemble spread (see ens_point below and DESIGN.md, K2).
__device__ __forceinline__ void ce2_packed(float& a0, float& a1, float& b0, float& b1) {
  const float l0 = fminf(a0, b0);
  const float l1 = fminf(a1, b1);
  b0 = __fsub_rn(__fadd_rn(a0, b0), l0);
  b1 = __fsub_rn(__fadd_rn(a1, b1), l1);
  a0 = l0;
  a1 = l1;
}
#define CE2(a, b) ce2_packed(v[a], v[(a) + 1], v[b], v[(b) + 1]);
#include "sort_networks.inc"
#undef CE
#undef CE2

constexpr int kEnsStats = 5;

// The packed network applies to full (unpadded), even-sized ensembles without
// NaN handling: padding is +inf and inf + inf - inf is NaN.
template <int MP, bool SKIPNA, bool EXACT>
constexpr bool kTwinSortOk = EXACT && !SKIPNA && MP >= 8 && MP % 2 == 0;

// Point-wise statistics of one grid point.  x[m] for m >= M is padding.
//   [0] skill_pt  = mean_m |t - x_m|                          (metrics.py:824)
//   [1] spread_pt = 2 * mean_m((2 r_m - M - 1) x_m) / (M - 1) (metrics.py:805-813)
//   [2] (t - xbar)^2          [3] var_m(x, ddof=1)     [4] [2] - [3] / M
// Every path sorts the mean-removed members; TWIN sorts them with the packed
// network, whose (a + b) - lo comparators round relative to the dispersion.
template <int MP, bool SKIPNA, bool EXACT, bool TWIN = false>
__device__ __forceinline__ void ens_point(float (&v)[MP], float t, int M, float (&val)[kEnsStats]) {
  static_assert(!TWIN || kTwinSortOk<MP, SKIPNA, EXACT>, "packed sort needs a full even ensemble");
  const float nanf_ = __int_as_float(0x7fc00000);
  const float inf_ = __int_as_float(0x7f800000);
  float sumx = 0.f, suma = 0.f;
  float nvalid = 0.f, navalid = 0.f;
#pragma unroll
  for (int m = 0; m < MP; ++m) {
    if (EXACT || m < M) {
      const float xm = v[m];
      const float a = fabsf(t - xm);  // metrics.py:824
      if (SKIPNA) {
        if (xm == xm) { sumx += xm; nvalid += 1.f; }
        if (a == a) { suma += a; navalid += 1.f; }
      } else {
        sumx += xm;
        suma += a;
      }
    }
  }
  const float fm = float(M);
  // Without skipna every division is by the constants M / M - 1: multiply by
  // their reciprocals (compile-time for a full ensemble) -- the IEEE division
  // is a ~15-instruction subroutine whose calls also fence the scheduler
  // (ens_pair_kernel gained 9 % from the same change); <= 1 ulp apart.
  const float inv_m = EXACT ? 1.f / float(MP) : 1.f / fm;
  const float inv_m1 = EXACT ? 1.f / float(MP > 1 ? MP - 1 : 1) : 1.f / (fm - 1.f);
  // __fmul_rn: the mean is rounded once and subtracted from every member; a
  // contracted x_m - sumx * inv_m would leave the residual of the rounded
  // reciprocal, so that equal members had a variance > 0.
  const float mean = SKIPNA ? sumx / nvalid : __fmul_rn(sumx, inv_m);  // 0/0 -> NaN like nanmean
  // The members are kept relative to the mean: the rank sum below is formed
  // on them, so its rounding scales with the ensemble's dispersion, not with
  // |x| (5e4 +- 5 would lose about three digits of the spread otherwise).  An
  // infinite or NaN mean (an infinite or, without skipna, NaN member) keeps
  // the raw members, whose rank sum is the reference's +-inf / NaN; the
  // variance is then NaN, like x - mean in the reference.
  const bool finite_mean = fabsf(mean) <= __int_as_float(0x7f7fffff);
  const float shift = finite_mean ? mean : 0.f;
  float ss = 0.f;
#pragma unroll
  for (int m = 0; m < MP; ++m) {
    if (EXACT || m < M) {
      const float dx = v[m] - shift;
      if (SKIPNA) {
        if (dx == dx) ss += dx * dx;
      } else {
        ss += dx * dx;
      }
      v[m] = dx;
    }
  }
  float var;
  if (!finite_mean) var = nanf_;
  else if (SKIPNA) var = nvalid > 1.f ? ss / (nvalid - 1.f) : nanf_;  // np.nanvar(ddof=1)
  else var = M > 1 ? ss * inv_m1 : ss / (fm - 1.f);                 // M == 1 -> 0/0 = NaN
  const float dm = t - mean;
  const float mse = dm * dm;
  val[0] = SKIPNA ? suma / navalid : suma * inv_m;
  val[2] = mse;
  val[3] = var;
  val[4] = mse - var * inv_m;  // metrics.py:564-565 (always divides by the full M)

  // ---- spread: ranks via sorting network (metrics.py:804-813) ---------------
  if (M < 2) {
    val[1] = 0.f;  // metrics.py:788-789
    return;
  }
#pragma unroll
  for (int m = 0; m < MP; ++m) {
    if (!EXACT && m >= M) v[m] = inf_;          // padding sorts last
    else if (SKIPNA && !(v[m] == v[m])) v[m] = inf_;  // NaN sorts last (np.argsort)
  }
  if constexpr (TWIN) SortNetTwin<MP>::run(v);
  else SortNet<MP>::run(v);
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < MP; ++i) {
    // coefficient 2 r - M - 1 with r = i + 1
    const float coef = float(2 * (i + 1)) - fm - 1.f;
    if (SKIPNA) {
      if (float(i) < nvalid) s += coef * v[i];
    } else if (EXACT || i < M) {
      s += coef * v[i];
    }
  }
  // The coefficients of the n valid ranks add up to n (n - M): 0 for a full
  // ensemble; under skipna with missing members the reference keeps M in
  // them, and the shift's share comes back here.
  if (SKIPNA) s += shift * (nvalid * (nvalid - fm));
  float spread = SKIPNA ? 2.f * (s / nvalid) * inv_m1 : 2.f * (s * inv_m) * inv_m1;
  if (!SKIPNA && !(sumx == sumx)) spread = nanf_;  // a NaN member poisons the point
  val[1] = spread;
}

}  // namespace wb2

// K4 fast path -- zonal energy spectrum as a prime-factor FFT on row pairs,
// rows staged by TMA (sm_90a).
//
// Replaces ZonalEnergySpectrum.compute (weatherbench2/derived_variables.py:
// 592-626) for the row lengths whose half N2 = N / 2 splits into three pairwise
// coprime radices RA * RB * RC (1440 longitudes: N2 = 720 = 9 * 16 * 5), plus
// the reductions that follow it in the callers: the time mean of
// scripts/compute_zonal_energy_spectrum.py:234 and (north star) the
// latitude-weighted meridional reduction with get_lat_weights
// (weatherbench2/metrics.py:40-60).
//
// Why this shape (the Stockham kernel of spectrum.cu is FMA-pipe bound, with
// as many integer index instructions as FP ones per butterfly):
//   * ROW PAIRS.  Two latitude rows (A, B) are transformed together: every
//     complex value is held as two 64-bit register pairs re = (re_A, re_B),
//     im = (im_A, im_B), loaded and stored as one 64-bit access, and every
//     operation is applied to both lanes -- the index arithmetic, shared-memory
//     instructions and twiddles are shared by two rows, and because the two
//     lanes are two independent rows there is not a single swizzle:
//     multiplying by -i is a register rename.
//   * PRIME-FACTOR (Good-Thomas) decomposition: with the input gathered by
//     n = (SA nA + SB nB + SC nC) mod N2 (S* = N2 / R*) and the output read at
//     k = (EA kA + EB kB + EC kC) mod N2 (E* the CRT idempotents), the N2-point
//     DFT is three plain DFTs of size RA, RB, RC along the axes of a
//     [RB][RA][RC] array: NO inter-stage twiddles (the Stockham version loaded
//     and multiplied 1 216 of them per row), IN PLACE (one shared buffer, no
//     ping-pong, no padding), and every index is a compile-time stride.
//   * The last stage computes butterfly (kA, kB) TOGETHER with its mirror
//     (-kA, -kB): bin p and bin N2 - p of the real-input split
//         X_p = (E + W_N^p O) / 2,  X_{N2-p} = conj(E - W_N^p O) / 2
//     are then both in the same thread's registers, so the power spectrum is
//     accumulated (over time steps, or over latitude rows with their weights)
//     straight from registers; the spectrum itself never goes to shared memory
//     unless it has to be written.
//   * TMA: the 2 G rows of the next work item are fetched by one elected thread
//     with cp.async.bulk (SASS UBLKCP) into a staging buffer guarded by an
//     mbarrier while stages B and C of the current item run.
//
// Work decomposition: a work item = G row pairs (2 G rows) of one field; a job
// = the items that share accumulators (mode 0: one item; mode 1: the same rows
// of every time step of a slot; mode 2: a chunk of row groups of every time
// step of a slot).  Persistent CTAs (the plan's MINB per SM) take jobs
// round-robin; the accumulators are flushed through shared memory (coalesced
// stores) at the end of a job.  Deterministic: no atomics, fixed summation
// order.
//
// Shared-memory traffic per row: one staging read, three in-place passes over
// the work array and the post twiddles.
#include <cmath>

#include "common.cuh"
#include "tma_utils.cuh"

namespace wb2 {
namespace pfa {

typedef unsigned long long u64;

// two complex numbers (lane 0 = row A, lane 1 = row B), split re / im
struct C2 {
  u64 re, im;
};

__device__ __forceinline__ u64 pk2(float lo, float hi) {
  u64 r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
  return r;
}
// same, but opaque to the optimiser: one pack per value (ptxas otherwise
// re-materialises the two MOVs at every use)
__device__ __forceinline__ u64 pk2v(float lo, float hi) {
  u64 r;
  asm volatile("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
  return r;
}
__device__ __forceinline__ u64 dup2(float c) { return pk2(c, c); }
__device__ __forceinline__ float lo2(u64 v) {
  float lo, hi;
  asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
  return lo;
}
__device__ __forceinline__ float hi2(u64 v) {
  float lo, hi;
  asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
  return hi;
}
// lane-wise arithmetic: two scalar round-to-nearest operations per pair (the
// __f*_rn intrinsics are never contracted, so mul + add stays two roundings)
__device__ __forceinline__ u64 add2(u64 a, u64 b) {
  return pk2(__fadd_rn(lo2(a), lo2(b)), __fadd_rn(hi2(a), hi2(b)));
}
__device__ __forceinline__ u64 sub2(u64 a, u64 b) {
  return pk2(__fsub_rn(lo2(a), lo2(b)), __fsub_rn(hi2(a), hi2(b)));
}
__device__ __forceinline__ u64 mul2(u64 a, u64 b) {
  return pk2(__fmul_rn(lo2(a), lo2(b)), __fmul_rn(hi2(a), hi2(b)));
}
__device__ __forceinline__ u64 fma2(u64 a, u64 b, u64 c) {
  return pk2(__fmaf_rn(lo2(a), lo2(b), lo2(c)), __fmaf_rn(hi2(a), hi2(b), hi2(c)));
}
// lane-wise c + a * s, leaving a lane alone whose s is 0: rows of zero weight
// (outside a latitude band, or the padding row of an odd nrow) contribute
// nothing, where 0 * inf or 0 * NaN would poison the sum
__device__ __forceinline__ u64 fma2_w(u64 a, u64 s, u64 c) {
  const float sl = lo2(s), sh = hi2(s);
  return pk2(sl == 0.f ? lo2(c) : __fmaf_rn(lo2(a), sl, lo2(c)),
             sh == 0.f ? hi2(c) : __fmaf_rn(hi2(a), sh, hi2(c)));
}
// the shift subtracted from a row before its transform: the row's first
// element, or 0 when that is not finite (inf - inf would turn the row into NaN)
__device__ __forceinline__ float row_shift(float x0) { return isfinite(x0) ? x0 : 0.f; }
__device__ __forceinline__ C2 cadd(C2 a, C2 b) { return {add2(a.re, b.re), add2(a.im, b.im)}; }
__device__ __forceinline__ C2 csub(C2 a, C2 b) { return {sub2(a.re, b.re), sub2(a.im, b.im)}; }
// a * (wr + i wi), wr / wi compile-time constants (they become FFMA immediates)
__device__ __forceinline__ C2 cmulc(C2 a, float wr, float wi) {
  C2 r;
  r.re = fma2(a.im, dup2(-wi), mul2(a.re, dup2(wr)));
  r.im = fma2(a.im, dup2(wr), mul2(a.re, dup2(wi)));
  return r;
}

template <int R>
__device__ __forceinline__ void dft(C2 (&v)[R]);

template <>
__device__ __forceinline__ void dft<1>(C2 (&)[1]) {}
template <>
__device__ __forceinline__ void dft<2>(C2 (&v)[2]) {
  const C2 a = v[0], b = v[1];
  v[0] = cadd(a, b);
  v[1] = csub(a, b);
}
template <>
__device__ __forceinline__ void dft<3>(C2 (&v)[3]) {
  constexpr float S = 0.86602540378443864676f;
  const C2 t = cadd(v[1], v[2]), d = csub(v[1], v[2]);
  const C2 m = {fma2(t.re, dup2(-0.5f), v[0].re), fma2(t.im, dup2(-0.5f), v[0].im)};
  v[0] = cadd(v[0], t);
  // n = -i S d = S (d.im, -d.re);  v1 = m + n, v2 = m - n
  v[1] = {fma2(d.im, dup2(S), m.re), fma2(d.re, dup2(-S), m.im)};
  v[2] = {fma2(d.im, dup2(-S), m.re), fma2(d.re, dup2(S), m.im)};
}
template <>
__device__ __forceinline__ void dft<4>(C2 (&v)[4]) {
  const C2 t0 = cadd(v[0], v[2]), t1 = csub(v[0], v[2]);
  const C2 t2 = cadd(v[1], v[3]), d = csub(v[1], v[3]);
  v[0] = cadd(t0, t2);
  v[2] = csub(t0, t2);
  v[1] = {add2(t1.re, d.im), sub2(t1.im, d.re)};  // t1 - i d
  v[3] = {sub2(t1.re, d.im), add2(t1.im, d.re)};  // t1 + i d
}
template <>
__device__ __forceinline__ void dft<5>(C2 (&v)[5]) {
  constexpr float c1 = 0.30901699437494742410f, c2 = -0.80901699437494742410f;
  constexpr float s1 = 0.95105651629515357212f, s2 = 0.58778525229247312917f;
  const C2 a = v[0];
  const C2 t1 = cadd(v[1], v[4]), t2 = cadd(v[2], v[3]);
  const C2 t3 = csub(v[1], v[4]), t4 = csub(v[2], v[3]);
  const C2 m1 = {fma2(t2.re, dup2(c2), fma2(t1.re, dup2(c1), a.re)),
                 fma2(t2.im, dup2(c2), fma2(t1.im, dup2(c1), a.im))};
  const C2 m2 = {fma2(t2.re, dup2(c1), fma2(t1.re, dup2(c2), a.re)),
                 fma2(t2.im, dup2(c1), fma2(t1.im, dup2(c2), a.im))};
  // u1 = s1 t3 + s2 t4, u2 = s2 t3 - s1 t4;  n = -i u = (u.im, -u.re)
  const C2 u1 = {fma2(t4.re, dup2(s2), mul2(t3.re, dup2(s1))),
                 fma2(t4.im, dup2(s2), mul2(t3.im, dup2(s1)))};
  const C2 u2 = {fma2(t4.re, dup2(-s1), mul2(t3.re, dup2(s2))),
                 fma2(t4.im, dup2(-s1), mul2(t3.im, dup2(s2)))};
  v[0] = cadd(a, cadd(t1, t2));
  v[1] = {add2(m1.re, u1.im), sub2(m1.im, u1.re)};
  v[4] = {sub2(m1.re, u1.im), add2(m1.im, u1.re)};
  v[2] = {add2(m2.re, u2.im), sub2(m2.im, u2.re)};
  v[3] = {sub2(m2.re, u2.im), add2(m2.im, u2.re)};
}

// cos / sin of 2 pi m / N for the composite radices (compile-time indices)
template <int N>
__device__ __forceinline__ float wcos(int m);
template <int N>
__device__ __forceinline__ float wsin(int m);
template <>
__device__ __forceinline__ float wcos<16>(int m) {
  constexpr float c[16] = {1.f, 0.92387953251128674f, 0.70710678118654752f,
                           0.38268343236508977f, 0.f, -0.38268343236508977f,
                           -0.70710678118654752f, -0.92387953251128674f, -1.f,
                           -0.92387953251128674f, -0.70710678118654752f,
                           -0.38268343236508977f, 0.f, 0.38268343236508977f,
                           0.70710678118654752f, 0.92387953251128674f};
  return c[m];
}
template <>
__device__ __forceinline__ float wsin<16>(int m) {
  constexpr float s[16] = {0.f, 0.38268343236508977f, 0.70710678118654752f,
                           0.92387953251128674f, 1.f, 0.92387953251128674f,
                           0.70710678118654752f, 0.38268343236508977f, 0.f,
                           -0.38268343236508977f, -0.70710678118654752f,
                           -0.92387953251128674f, -1.f, -0.92387953251128674f,
                           -0.70710678118654752f, -0.38268343236508977f};
  return s[m];
}
template <>
__device__ __forceinline__ float wcos<9>(int m) {
  constexpr float c[9] = {1.f, 0.76604444311897804f, 0.17364817766693035f, -0.5f,
                          -0.93969262078590838f, -0.93969262078590838f, -0.5f,
                          0.17364817766693035f, 0.76604444311897804f};
  return c[m];
}
template <>
__device__ __forceinline__ float wsin<9>(int m) {
  constexpr float s[9] = {0.f, 0.64278760968653933f, 0.98480775301220806f,
                          0.86602540378443865f, 0.34202014332566873f,
                          -0.34202014332566873f, -0.86602540378443865f,
                          -0.98480775301220806f, -0.64278760968653933f};
  return s[m];
}
template <>
__device__ __forceinline__ float wcos<8>(int m) {
  constexpr float c[8] = {1.f, 0.70710678118654752f, 0.f, -0.70710678118654752f,
                          -1.f, -0.70710678118654752f, 0.f, 0.70710678118654752f};
  return c[m];
}
template <>
__device__ __forceinline__ float wsin<8>(int m) {
  constexpr float s[8] = {0.f, 0.70710678118654752f, 1.f, 0.70710678118654752f,
                          0.f, -0.70710678118654752f, -1.f, -0.70710678118654752f};
  return s[m];
}

// Cooley-Tukey composite of size R1 * R2 in registers:
//   input n = R2 n1 + n2, output k = k1 + R1 k2, twiddle exp(-2 pi i n2 k1 / N)
template <int R1, int R2>
__device__ __forceinline__ void dft_composite(C2 (&v)[R1 * R2]) {
  constexpr int N = R1 * R2;
  C2 y[R2][R1];
#pragma unroll
  for (int n2 = 0; n2 < R2; ++n2) {
    C2 col[R1];
#pragma unroll
    for (int n1 = 0; n1 < R1; ++n1) col[n1] = v[R2 * n1 + n2];
    dft<R1>(col);
#pragma unroll
    for (int k1 = 0; k1 < R1; ++k1) {
      const int m = (n2 * k1) % N;
      if (m == 0) {
        y[n2][k1] = col[k1];
      } else if (4 * m == N) {  // times -i: a rename plus one sign flip (ALU pipe)
        y[n2][k1] = {col[k1].im, col[k1].re ^ 0x8000000080000000ull};
      } else {
        y[n2][k1] = cmulc(col[k1], wcos<N>(m), -wsin<N>(m));
      }
    }
  }
#pragma unroll
  for (int k1 = 0; k1 < R1; ++k1) {
    C2 row[R2];
#pragma unroll
    for (int n2 = 0; n2 < R2; ++n2) row[n2] = y[n2][k1];
    dft<R2>(row);
#pragma unroll
    for (int k2 = 0; k2 < R2; ++k2) v[k1 + R1 * k2] = row[k2];
  }
}
template <>
__device__ __forceinline__ void dft<16>(C2 (&v)[16]) { dft_composite<4, 4>(v); }
template <>
__device__ __forceinline__ void dft<9>(C2 (&v)[9]) { dft_composite<3, 3>(v); }
template <>
__device__ __forceinline__ void dft<8>(C2 (&v)[8]) { dft_composite<4, 2>(v); }

// ---------------------------------------------------------------------------
constexpr int idem(int n2, int r) {  // CRT idempotent: 1 mod r, 0 mod n2 / r
  const int m = n2 / r;
  int x = m;
  while (x % r != 1 % r) x += m;
  return x % n2;
}

template <int RA_, int RB_, int RC_, int G_, int NT_, int MINB_ = 2>
struct Plan {
  static constexpr int RA = RA_, RB = RB_, RC = RC_, G = G_, NT = NT_, MINB = MINB_;
  static constexpr int N2 = RA * RB * RC, NK = N2 + 1, N = 2 * N2;
  static constexpr int SA = N2 / RA, SB = N2 / RB, SC = N2 / RC;  // Good's input map
  static constexpr int EA = idem(N2, RA), EB = idem(N2, RB), EC = idem(N2, RC);
  static constexpr int LB = RA * RC, LA = RC;  // in-place layout [RB][RA][RC]
  static constexpr int NTA = RB * RC, NTB = RA * RC;  // tasks per row pair
  // mirrored pairs {(kA, kB), (-kA, -kB)}: the self-paired ones are kA = 0
  // (RA odd) with kB = 0 and, for even RB, kB = RB / 2
  static constexpr int NSELF = (RA % 2 == 0 ? 2 : 1) * (RB % 2 == 0 ? 2 : 1);
  static constexpr int NTC = (RA * RB - NSELF) / 2 + NSELF;
  static constexpr int kRowBytes = N * 4;
  static constexpr int kStageBytes = 2 * G * kRowBytes;
  static constexpr int kWorkBytes = G * N2 * 16;
  static constexpr int kTwnBytes = N2 * 16;
  static constexpr int kTaskBytes = ((NTC * 16 + 127) / 128) * 128;
  // + the mbarrier (16 B) and the 2 G row shifts
  static constexpr int kSmem = kStageBytes + kWorkBytes + kTwnBytes + kTaskBytes + 64 + 8 * G;
  // thread slots per row pair, padded to half-warps so that the 64-bit shared
  // accesses of a half-warp stay inside one row pair (conflict-free strides)
  static constexpr int PTB = (NTB + 15) / 16 * 16, PTC = (NTC + 15) / 16 * 16;
  static_assert(G * PTC <= NT, "stage C keeps one task per thread (register accumulators)");
  static_assert(G * NTA <= NT && G * PTB <= NT, "one task per thread in every stage");
  static_assert(2 * G * NK * 4 <= kWorkBytes, "flush tile must fit the work buffer");
  static_assert(N2 % 2 == 0, "rows must be multiples of 16 bytes for TMA");
};

struct Params {
  const float* x;       // [nfield][nrow][N]
  float* out;           // modes 0/1: [nslot][nrow][NK];  mode 2: partial [njob][NK]
  const float4* twn;    // [N2] (wr, wr, wi, wi) of exp(-2 pi i p / N)
  const int4* ctask;    // [NTC] {offset of (kA,kB), offset of its mirror, k0, self}
  const float* scale;   // [2 G ngroup] per-row factor, 0 beyond nrow
  int64_t nslot;        // output slots (fields are slot-minor: field = ti * nslot + slot)
  int32_t ntimes;       // fields per slot
  int32_t nrow;
  int32_t ngroup;       // groups of G row pairs per field
  int32_t gpc;          // groups per chunk (1 in modes 0 / 1)
  int32_t nchunk;       // chunks per field
  int64_t njob;         // nslot * nchunk
  int32_t mode;         // 0 store, 1 add to out, 2 latitude-reduced partials
};

// position in the job / item sequence of one CTA (uniform across the CTA)
struct Cursor {
  int64_t job;
  int32_t ti, gi, gbeg, gend;
  int64_t slot;
  __device__ __forceinline__ void open(const Params& p) {
    if (job < p.njob) {
      slot = job / p.nchunk;
      const int chunk = static_cast<int>(job - slot * p.nchunk);
      gbeg = chunk * p.gpc;
      gend = min(p.ngroup, gbeg + p.gpc);
      gi = gbeg;
      ti = 0;
    }
  }
  __device__ __forceinline__ bool valid(const Params& p) const { return job < p.njob; }
  __device__ __forceinline__ bool last_of_job(const Params& p) const {
    return gi == gend - 1 && ti == p.ntimes - 1;
  }
  __device__ __forceinline__ void advance(const Params& p) {
    if (++gi == gend) {
      gi = gbeg;
      if (++ti == p.ntimes) {
        job += gridDim.x;
        open(p);
      }
    }
  }
};

template <class P>
__device__ __forceinline__ void issue_item(const Params& p, const Cursor& c, float* staging,
                                           uint64_t* bar) {
  const int64_t field = int64_t(c.ti) * p.nslot + c.slot;
  const float* base = p.x + field * p.nrow * int64_t(P::N);
  mbar_arrive_expect_tx(bar, P::kStageBytes);
#pragma unroll 1
  for (int r = 0; r < 2 * P::G; ++r) {
    const int row = min(2 * P::G * c.gi + r, p.nrow - 1);  // padding rows repeat the last row
    tma_load_1d(staging + r * P::N, base + int64_t(row) * P::N, P::kRowBytes, bar);
  }
}

template <class P, int MODE>
__global__ void __launch_bounds__(P::NT, P::MINB) spectrum_pfa_kernel(const Params p) {
  constexpr int RA = P::RA, RB = P::RB, RC = P::RC, G = P::G, NT = P::NT;
  constexpr int N2 = P::N2, NK = P::NK;
  extern __shared__ __align__(128) unsigned char smem[];
  float* staging = reinterpret_cast<float*>(smem);
  // in-place work array, planar: re and im as separate 64-bit planes (an
  // interleaved 128-bit element would need its four registers adjacent, which
  // costs four MOVs per store)
  u64* const work_re = reinterpret_cast<u64*>(smem + P::kStageBytes);
  u64* const work_im = work_re + G * N2;
  const ulonglong2* twn =
      reinterpret_cast<const ulonglong2*>(smem + P::kStageBytes + P::kWorkBytes);
  const int4* ctask = reinterpret_cast<const int4*>(smem + P::kStageBytes + P::kWorkBytes +
                                                     P::kTwnBytes);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + P::kStageBytes + P::kWorkBytes +
                                               P::kTwnBytes + P::kTaskBytes);
  float* const shift = reinterpret_cast<float*>(full + 2);  // [2 G] of the current item
  float* const tile = reinterpret_cast<float*>(work_re);  // flush tile [2 G][NK], aliases `work`
  const int tid = threadIdx.x;

  {
    float4* d = reinterpret_cast<float4*>(smem + P::kStageBytes + P::kWorkBytes);
    for (int i = tid; i < N2; i += NT) d[i] = p.twn[i];
    int4* t = reinterpret_cast<int4*>(smem + P::kStageBytes + P::kWorkBytes + P::kTwnBytes);
    for (int i = tid; i < P::NTC; i += NT) t[i] = p.ctask[i];
  }
  Cursor cur;
  cur.job = blockIdx.x;
  cur.open(p);
  if (tid == 0) {
    mbar_init(full, 1);
    mbar_fence_init();
    if (cur.valid(p)) issue_item<P>(p, cur, staging, full);
  }
  __syncthreads();

  // ---- thread-invariant task geometry --------------------------------------
  // stage A (radix RA, staging -> work): half-warps share nC and span nB, so the
  // gathered LDS.64 hit 16 distinct bank pairs (SB is odd)
  const bool a_on = tid < G * P::NTA;
  int a_e0 = 0, a_src = 0, a_dst = 0, a_g = 0;
  {
    const int g = tid / P::NTA, r = tid - g * P::NTA;
    const int nC = r / RB, nB = r - nC * RB;
    a_e0 = (P::SB * nB + P::SC * nC) % N2;
    a_src = 2 * g * N2;  // float2 index of row A of the pair; row B follows at + N2
    a_dst = g * N2 + nB * P::LB + nC;
    a_g = g;
  }
  // stage B (radix RB, in place): consecutive threads, consecutive elements
  bool b_on;
  int b_off = 0;
  {
    const int g = tid / P::PTB, r = tid - g * P::PTB;
    b_on = g < G && r < P::NTB;
    b_off = g * N2 + r;
  }
  // stage C (radix RC on a butterfly and its mirror, then the real-input split)
  int c_g = tid / P::PTC, c_off1 = 0, c_off2 = 0, c_k0 = 0, c_self = 0;  // c_k0 == 0: owns bin 0
  const bool c_on = c_g < G && tid - c_g * P::PTC < P::NTC;
  if (c_on) {
    const int4 t = ctask[tid - c_g * P::PTC];
    c_off1 = c_g * N2 + t.x;
    c_off2 = c_g * N2 + t.y;
    c_k0 = t.z;
    c_self = t.w;
  }
  u64 acc_a[RC], acc_b[RC];
#pragma unroll
  for (int i = 0; i < RC; ++i) acc_a[i] = acc_b[i] = 0ull;

  uint32_t parity = 0;
  while (cur.valid(p)) {
    Cursor nxt = cur;
    nxt.advance(p);
    mbar_wait(full, parity);
    parity ^= 1u;

    // ---- stage A --------------------------------------------------------------
    if (a_on) {
      const float2* ra = reinterpret_cast<const float2*>(staging) + a_src;
      const float2* rb = ra + N2;
      // transform x - s (s = the row's first element): the DFT is shift-invariant
      // except for bin 0, and the butterflies now round relative to the row's
      // variation instead of its mean; stage C adds N s back to bin 0
      const float sa = row_shift(ra[0].x), sb = row_shift(rb[0].x);
      if (a_e0 == 0) {
        shift[2 * a_g] = sa;
        shift[2 * a_g + 1] = sb;
      }
      C2 v[RA];
#pragma unroll
      for (int nA = 0; nA < RA; ++nA) {
        int e = a_e0 + P::SA * nA;
        e = e >= N2 ? e - N2 : e;
        const float2 a = ra[e], b = rb[e];
        v[nA].re = pk2v(__fsub_rn(a.x, sa), __fsub_rn(b.x, sb));
        v[nA].im = pk2v(__fsub_rn(a.y, sa), __fsub_rn(b.y, sb));
      }
      dft<RA>(v);
#pragma unroll
      for (int kA = 0; kA < RA; ++kA) {
        work_re[a_dst + kA * P::LA] = v[kA].re;
        work_im[a_dst + kA * P::LA] = v[kA].im;
      }
    }
    __syncthreads();  // staging consumed, work complete
    if (tid == 0 && nxt.valid(p)) issue_item<P>(p, nxt, staging, full);

    // ---- stage B --------------------------------------------------------------
    if (b_on) {
      C2 v[RB];
#pragma unroll
      for (int nB = 0; nB < RB; ++nB)
        v[nB] = {work_re[b_off + nB * P::LB], work_im[b_off + nB * P::LB]};
      dft<RB>(v);
#pragma unroll
      for (int kB = 0; kB < RB; ++kB) {
        work_re[b_off + kB * P::LB] = v[kB].re;
        work_im[b_off + kB * P::LB] = v[kB].im;
      }
    }
    __syncthreads();

    // ---- stage C + split + power ---------------------------------------------
    if (c_on) {
      C2 b1[RC], b2[RC];
#pragma unroll
      for (int i = 0; i < RC; ++i) {
        b1[i] = {work_re[c_off1 + i], work_im[c_off1 + i]};
        b2[i] = {work_re[c_off2 + i], work_im[c_off2 + i]};
      }
      dft<RC>(b1);
      dft<RC>(b2);
      // 2 N s for the thread that owns bin 0 (the split computes 2 X_p), else 0
      u64 dc = 0ull;
      if (c_k0 == 0)
        dc = pk2(__fmul_rn(float(2 * P::N), shift[2 * c_g]),
                 __fmul_rn(float(2 * P::N), shift[2 * c_g + 1]));
      u64 scl = 0ull;
      if (MODE == 2) {
        const int row = 2 * (G * cur.gi + c_g);
        scl = pk2(__ldg(p.scale + row), __ldg(p.scale + row + 1));
      }
#pragma unroll
      for (int kC = 0; kC < RC; ++kC) {
        int pbin = c_k0 + (kC * P::EC) % N2;
        pbin = pbin >= N2 ? pbin - N2 : pbin;
        const ulonglong2 w = twn[pbin];  // (wr, wr), (wi, wi)
        const C2 zp = b1[kC], zq = b2[(RC - kC) % RC];
        const u64 e_re = add2(zp.re, zq.re), e_im = sub2(zp.im, zq.im);
        const u64 d_re = sub2(zp.re, zq.re), d_im = add2(zp.im, zq.im);
        // W (-i D):  re = wr d_im + wi d_re,  im = wi d_im - wr d_re
        const u64 t1 = fma2(w.y, d_re, mul2(w.x, d_im));
        const u64 t2 = sub2(mul2(w.x, d_re), mul2(w.y, d_im));  // = -im
        u64 xa_re = add2(e_re, t1);
        const u64 xa_im = sub2(e_im, t2);
        if (kC == 0) xa_re = add2(xa_re, dc);  // bin c_k0: the shift back into bin 0
        const u64 xb_re = sub2(e_re, t1), xb_im = add2(e_im, t2);
        if (MODE == 2) {
          const u64 pa = fma2(xa_im, xa_im, mul2(xa_re, xa_re));
          const u64 pb = fma2(xb_im, xb_im, mul2(xb_re, xb_re));
          acc_a[kC] = fma2_w(pa, scl, acc_a[kC]);
          acc_b[kC] = fma2_w(pb, scl, acc_b[kC]);
        } else {
          acc_a[kC] = fma2(xa_im, xa_im, fma2(xa_re, xa_re, acc_a[kC]));
          acc_b[kC] = fma2(xb_im, xb_im, fma2(xb_re, xb_re, acc_b[kC]));
        }
      }
    }

    if (cur.last_of_job(p)) {
      __syncthreads();  // everyone is done reading `work`; it becomes the tile
      if (c_on) {
        float* ta = tile + (2 * c_g) * NK;
        float* tb = ta + NK;
        // modes 0 / 1: the per-row factor is applied here, so that the copy-out
        // below is a flat, unrolled add (mode 2 applied it per item already)
        float sa = 1.f, sb = 1.f;
        if (MODE != 2) {
          const int row = 2 * (G * cur.gi + c_g);
          sa = __ldg(p.scale + row);
          sb = __ldg(p.scale + row + 1);
        }
#pragma unroll
        for (int kC = 0; kC < RC; ++kC) {
          int pbin = c_k0 + (kC * P::EC) % N2;
          pbin = pbin >= N2 ? pbin - N2 : pbin;
          const bool va = !c_self || kC <= (RC - kC) % RC;
          const bool vb = va && (2 * pbin != N2);
          const float h0 = pbin == 0 ? 0.5f : 1.f;  // c_k = 1 for the zonal mean
          if (va) {
            ta[pbin] = lo2(acc_a[kC]) * (sa * h0);
            tb[pbin] = hi2(acc_a[kC]) * (sb * h0);
          }
          if (vb) {
            ta[N2 - pbin] = lo2(acc_b[kC]) * sa;
            tb[N2 - pbin] = hi2(acc_b[kC]) * sb;
          }
          acc_a[kC] = acc_b[kC] = 0ull;
        }
      }
      __syncthreads();
      if (MODE == 2) {
        // rows already carry their weights: add the 2 G rows in a fixed order
        float* o = p.out + cur.job * NK;
        for (int k = tid; k < NK; k += NT) {
          float s = 0.f;
#pragma unroll
          for (int r = 0; r < 2 * G; ++r) s += tile[r * NK + k];
          o[k] = s;
        }
      } else {
        // the rows of a group are contiguous in `out`: one flat range; loads of
        // the read-modify-write are issued kU at a time (the un-unrolled loop
        // held a third of the kernel's stall samples on the first FFMA)
        const int row0 = 2 * G * cur.gi;
        const int n = min(2 * G, p.nrow - row0) * NK;
        float* o = p.out + (cur.slot * p.nrow + row0) * int64_t(NK);
        constexpr int kU = 6;
        for (int i0 = tid; i0 < n; i0 += kU * NT) {
          float v[kU];
#pragma unroll
          for (int u = 0; u < kU; ++u) {
            const int i = i0 + u * NT;
            v[u] = (MODE == 1 && i < n) ? o[i] : 0.f;
          }
#pragma unroll
          for (int u = 0; u < kU; ++u) {
            const int i = i0 + u * NT;
            if (i < n) o[i] = v[u] + tile[i];
          }
        }
      }
    }
    __syncthreads();  // the work buffer (and the tile in it) is overwritten by the next stage A
    cur = nxt;
  }
}

// sums the per-chunk partials of mode 2 in a fixed order
__global__ void latsum_finalize_kernel(const float* __restrict__ partial, float* __restrict__ out,
                                       int64_t nslot, int nchunk, int nk, int accumulate) {
  const int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
  if (i >= nslot * nk) return;
  const int64_t slot = i / nk;
  const int k = static_cast<int>(i - slot * nk);
  float s = 0.f;
  for (int c = 0; c < nchunk; ++c) s += partial[(slot * nchunk + c) * nk + k];
  out[i] = accumulate ? out[i] + s : s;
}

template <class P>
static void build_tables(std::vector<float4>* twn, std::vector<int4>* ctask) {
  const double two_pi = 6.283185307179586476925286766559;
  twn->resize(P::N2);
  for (int k = 0; k < P::N2; ++k) {
    const double a = -two_pi * k / P::N;
    const float wr = static_cast<float>(cos(a)), wi = static_cast<float>(sin(a));
    (*twn)[k] = make_float4(wr, wr, wi, wi);
  }
  ctask->clear();
  std::vector<char> seen(P::RA * P::RB, 0);
  // kA = 1, 2, ... first: their kB runs are whole half-warps (16 consecutive kB
  // hit 16 distinct bank pairs because LB is odd); the shorter kA = 0 run last
  for (int ia = 1; ia <= P::RA; ++ia)
    for (int kB = 0; kB < P::RB; ++kB) {
      const int kA = ia % P::RA;
      if (seen[kA * P::RB + kB]) continue;
      const int qA = (P::RA - kA) % P::RA, qB = (P::RB - kB) % P::RB;
      seen[kA * P::RB + kB] = 1;
      seen[qA * P::RB + qB] = 1;
      int4 t;
      t.x = kB * P::LB + kA * P::LA;
      t.y = qB * P::LB + qA * P::LA;
      t.z = (kA * P::EA + kB * P::EB) % P::N2;
      t.w = (qA == kA && qB == kB) ? 1 : 0;
      ctask->push_back(t);
    }
}

template <class P>
static int launch(wb2_ctx* ctx, const float* x, int64_t nfield, int32_t nrow,
                  const double* scale, float* out, int mode, int64_t nslot) {
  const int latsum_accumulate = mode == 3;  // mode 3 = mode 2 adding to `out`
  if (mode == 3) mode = 2;
  std::vector<float4> twn;
  std::vector<int4> ctask;
  build_tables<P>(&twn, &ctask);
  if (static_cast<int>(ctask.size()) != P::NTC) {
    set_error("spectrum_pfa: task table has %zu entries, expected %d", ctask.size(), P::NTC);
    return WB2_EINVAL;
  }
  Params p;
  p.x = x;
  p.nslot = nslot;
  p.ntimes = static_cast<int32_t>(nfield / nslot);
  p.nrow = nrow;
  const int npair = (nrow + 1) / 2;
  p.ngroup = (npair + P::G - 1) / P::G;
  p.mode = mode;
  // latitude chunks of mode 2: enough jobs to fill the machine, few partials
  const int64_t want_jobs = int64_t(ctx->num_sms) * P::MINB * 4;
  if (mode == 2) {
    int nchunk = static_cast<int>((want_jobs + nslot - 1) / nslot);
    if (nchunk < 1) nchunk = 1;
    if (nchunk > p.ngroup) nchunk = p.ngroup;
    p.gpc = (p.ngroup + nchunk - 1) / nchunk;
    p.nchunk = (p.ngroup + p.gpc - 1) / p.gpc;
  } else {
    p.gpc = 1;
    p.nchunk = p.ngroup;
  }
  p.njob = nslot * p.nchunk;
  // per-row factor: circumference / N^2 (rfft norm='forward') * 2 (c_k; bin 0 is
  // halved at the flush) / 4 (the split computes 2 X_p): scale / (2 N^2)
  std::vector<float> sc(size_t(2) * P::G * p.ngroup, 0.f);
  for (int i = 0; i < nrow; ++i)
    sc[i] = static_cast<float>(scale[i] / (2.0 * double(P::N) * double(P::N)));

  Packer pk(ctx);
  const size_t o1 = pk.add(twn.data(), twn.size() * sizeof(float4));
  const size_t o2 = pk.add(ctask.data(), ctask.size() * sizeof(int4));
  const size_t o3 = pk.add(sc.data(), sc.size() * sizeof(float));
  size_t o4 = 0;
  if (mode == 2) o4 = pk.reserve(size_t(p.njob) * P::NK * sizeof(float));
  WB2_TRY(pk.commit());
  p.twn = pk.dev<float4>(o1);
  p.ctask = pk.dev<int4>(o2);
  p.scale = pk.dev<float>(o3);
  p.out = mode == 2 ? pk.dev<float>(o4) : out;

  const int64_t max_cta = int64_t(ctx->num_sms) * P::MINB;
  const unsigned grid = static_cast<unsigned>(p.njob < max_cta ? p.njob : max_cta);
  auto kernel = mode == 0 ? spectrum_pfa_kernel<P, 0>
                          : (mode == 1 ? spectrum_pfa_kernel<P, 1> : spectrum_pfa_kernel<P, 2>);
  WB2_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    P::kSmem));
  kernel<<<grid, P::NT, P::kSmem, ctx->stream>>>(p);
  WB2_CUDA_TRY(cudaGetLastError());
  ctx->launches += 1;
  if (mode == 2) {
    const int64_t n = nslot * P::NK;
    latsum_finalize_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, ctx->stream>>>(
        p.out, out, nslot, p.nchunk, P::NK, latsum_accumulate);
    WB2_CUDA_TRY(cudaGetLastError());
    ctx->launches += 1;
  }
  WB2_TRY(pk.release());
  return WB2_OK;
}

}  // namespace pfa

// Returns 1 when the prime-factor kernel handled the call, 0 when the shape /
// alignment is not eligible (the caller falls back), < 0 on error.
//   mode 0: out[field][row][k] = S;   mode 1: out[slot][row][k] += sum_time S;
//   mode 2: out[slot][k] = sum_time sum_row scale[row] * S-without-circumference
//           (`scale` already holds circumference * row weight);  mode 3: same,
//           added to `out`.
int spectrum_pfa_try(wb2_ctx* ctx, const float* x, int64_t nfield, int32_t nrow, int32_t ncol,
                     const double* scale, float* out, int mode, int64_t nslot) {
  const char* force = getenv("WB2_SPECTRUM_PATH");
  if (force && strcmp(force, "pfa") != 0) return 0;
  if ((reinterpret_cast<uintptr_t>(x) & 15) != 0) return 0;
  if (nrow < 1 || nfield < 1 || nslot < 1 || nfield % nslot != 0) return 0;
  int rc;
  switch (ncol) {
    // 3 CTAs of 5 warps per SM: fastest on H100 in every mode (DESIGN.md, K4)
    case 1440: rc = pfa::launch<pfa::Plan<9, 16, 5, 2, 160, 3>>(ctx, x, nfield, nrow, scale, out,
                                                                 mode, nslot); break;
    case 720: rc = pfa::launch<pfa::Plan<9, 8, 5, 5, 256>>(ctx, x, nfield, nrow, scale, out,
                                                            mode, nslot); break;
    case 240: rc = pfa::launch<pfa::Plan<3, 8, 5, 6, 256>>(ctx, x, nfield, nrow, scale, out,
                                                            mode, nslot); break;
    default: return 0;
  }
  return rc == WB2_OK ? 1 : rc;
}

}  // namespace wb2

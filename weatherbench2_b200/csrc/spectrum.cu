// K4 -- zonal energy spectrum (sm_90a).
//
// Replaces ZonalEnergySpectrum.compute (weatherbench2/derived_variables.py:
// 592-626):  F = rfft(x, axis=lon, norm='forward');  S_k = |F_k|^2 * (1 if k == 0
// else 2) (the Nyquist bin is doubled too, :600);  S *= circumference(lat) (:626).
// Optionally sums over time on the device, which is what the driver script does
// right after (xbeam.Mean(['time']), scripts/compute_zonal_energy_spectrum.py:234).
//
// Algorithm: a real FFT of length N = 2 * N2 per latitude row as one complex
// FFT of length N2 (z_j = x_2j + i x_2j+1, i.e. the row read as float2) plus the
// standard split post-pass.  The complex FFT is a Stockham autosort FFT in
// shared memory with register butterflies of radix 16, 9, 8, 5, 4, 3, 2
// (N2 = 720 = 16 * 9 * 5 for 1440 longitudes: three passes); radix 16 / 9 / 8
// are Cooley-Tukey composites of the 4 / 3 / 2 butterflies with compile-time
// twiddles.  The first stage reads straight from HBM (coalesced float2); the
// post-pass multiplies |X_k|^2 by c_k * scale[row] / N^2 and either writes or
// accumulates in registers over the time loop (deterministic: a CTA owns its
// output rows and walks time in order).  Stage twiddles come from a
// double-precision host table rounded to float32, staged in shared memory.
// Shared arrays are padded by one float2 every 16 so that the stride-R writes
// of the first stage are 2-way instead of 16-way bank conflicts; (row, j)
// decoding uses multiply-high division.
//
// Roofline: HBM, 4 B read per cell (+ 2 B written when per-time spectra are
// kept); at N = 1440 the FFT's ~30 flop-instructions per cell are close to the
// FP32 ridge of the chip (DESIGN.md).
#include <cmath>

#include "common.cuh"

namespace wb2 {

constexpr int kSpThreads = 256;
constexpr int kSpMaxStages = 16;
constexpr int kSpMaxAcc = 24;
constexpr int kSpMaxRows = 32;  // rows per CTA
// static shared memory of the kernels (the per-row shifts): counts towards the
// 48 KB a launch may use without opting in
constexpr size_t kSpStaticSmem = kSpMaxRows * sizeof(float);

struct SpecParams {
  const float* x;
  float* out;
  const float2* tw2;   // W_N2^k, k = 0..N2-1
  const float2* twn;   // W_N^k,  k = 0..N2
  const float* scale;  // [nrow]  circumference / N^2
  int64_t nfield_out;
  int32_t ntimes;
  int32_t nrow, n, n2, nk;
  int32_t rows_per_block, nblk;
  int32_t nstage;
  int32_t radix[kSpMaxStages];
  int32_t accumulate;
  int32_t row_pitch;  // padded float2 per row in shared memory
};

__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}
__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
// multiply by -i:  (x, y) -> (y, -x)
__device__ __forceinline__ float2 mul_mi(float2 a) { return make_float2(a.y, -a.x); }
// padded shared-memory index
__device__ __forceinline__ int pad(int i) { return i + (i >> 4); }
// floor(x / d) for 0 <= x < 2^20 via multiply-high; m = ceil(2^32 / d)
__device__ __forceinline__ int fast_div(int x, unsigned m, int d) {
  return d == 1 ? x : static_cast<int>(__umulhi(static_cast<unsigned>(x), m));
}
// The shift subtracted from a row before its transform: the row's first element
// (0 when that is not finite: inf - inf would turn the row into NaN).  The DFT
// is shift-invariant except for bin 0, so the butterflies round relative to
// the row's variation instead of its mean; the post-pass adds N s back to X_0.
__device__ __forceinline__ float row_shift(const float2* row) {
  const float s = __ldg(reinterpret_cast<const float*>(row));
  return isfinite(s) ? s : 0.f;
}
static unsigned magic(int d) {
  return d <= 1 ? 0u : static_cast<unsigned>(((1ull << 32) + d - 1) / d);
}

template <int R> __device__ __forceinline__ void dft(float2 (&v)[R]);

template <> __device__ __forceinline__ void dft<1>(float2 (&)[1]) {}
template <> __device__ __forceinline__ void dft<2>(float2 (&v)[2]) {
  const float2 a = v[0], b = v[1];
  v[0] = cadd(a, b);
  v[1] = csub(a, b);
}
template <> __device__ __forceinline__ void dft<3>(float2 (&v)[3]) {
  const float s = 0.86602540378443864676f;
  const float2 a = v[0], t1 = cadd(v[1], v[2]), d = csub(v[1], v[2]);
  const float2 m = make_float2(a.x - 0.5f * t1.x, a.y - 0.5f * t1.y);
  const float2 n = make_float2(s * d.y, -s * d.x);  // -i * s * d
  v[0] = cadd(a, t1);
  v[1] = cadd(m, n);
  v[2] = csub(m, n);
}
template <> __device__ __forceinline__ void dft<4>(float2 (&v)[4]) {
  const float2 t0 = cadd(v[0], v[2]), t1 = csub(v[0], v[2]);
  const float2 t2 = cadd(v[1], v[3]), t3 = mul_mi(csub(v[1], v[3]));
  v[0] = cadd(t0, t2);
  v[2] = csub(t0, t2);
  v[1] = cadd(t1, t3);
  v[3] = csub(t1, t3);
}
template <> __device__ __forceinline__ void dft<5>(float2 (&v)[5]) {
  const float c1 = 0.30901699437494742410f, c2 = -0.80901699437494742410f;
  const float s1 = 0.95105651629515357212f, s2 = 0.58778525229247312917f;
  const float2 a = v[0];
  const float2 t1 = cadd(v[1], v[4]), t2 = cadd(v[2], v[3]);
  const float2 t3 = csub(v[1], v[4]), t4 = csub(v[2], v[3]);
  const float2 m1 = make_float2(a.x + c1 * t1.x + c2 * t2.x, a.y + c1 * t1.y + c2 * t2.y);
  const float2 m2 = make_float2(a.x + c2 * t1.x + c1 * t2.x, a.y + c2 * t1.y + c1 * t2.y);
  const float2 n1 = mul_mi(make_float2(s1 * t3.x + s2 * t4.x, s1 * t3.y + s2 * t4.y));
  const float2 n2 = mul_mi(make_float2(s2 * t3.x - s1 * t4.x, s2 * t3.y - s1 * t4.y));
  v[0] = cadd(a, cadd(t1, t2));
  v[1] = cadd(m1, n1);
  v[4] = csub(m1, n1);
  v[2] = cadd(m2, n2);
  v[3] = csub(m2, n2);
}

// cos / sin of 2 pi m / N for the composite radices (compile-time indices)
template <int N> struct Wc;
template <> struct Wc<16> {
  static __device__ __forceinline__ float2 w(int m) {
    constexpr float c[16] = {1.f, 0.92387953251128674f, 0.70710678118654752f,
                             0.38268343236508977f, 0.f, -0.38268343236508977f,
                             -0.70710678118654752f, -0.92387953251128674f, -1.f,
                             -0.92387953251128674f, -0.70710678118654752f,
                             -0.38268343236508977f, 0.f, 0.38268343236508977f,
                             0.70710678118654752f, 0.92387953251128674f};
    constexpr float s[16] = {0.f, 0.38268343236508977f, 0.70710678118654752f,
                             0.92387953251128674f, 1.f, 0.92387953251128674f,
                             0.70710678118654752f, 0.38268343236508977f, 0.f,
                             -0.38268343236508977f, -0.70710678118654752f,
                             -0.92387953251128674f, -1.f, -0.92387953251128674f,
                             -0.70710678118654752f, -0.38268343236508977f};
    return make_float2(c[m], -s[m]);  // forward transform: exp(-2 pi i m / N)
  }
};
template <> struct Wc<9> {
  static __device__ __forceinline__ float2 w(int m) {
    constexpr float c[9] = {1.f, 0.76604444311897804f, 0.17364817766693035f, -0.5f,
                            -0.93969262078590838f, -0.93969262078590838f, -0.5f,
                            0.17364817766693035f, 0.76604444311897804f};
    constexpr float s[9] = {0.f, 0.64278760968653933f, 0.98480775301220806f,
                            0.86602540378443865f, 0.34202014332566873f,
                            -0.34202014332566873f, -0.86602540378443865f,
                            -0.98480775301220806f, -0.64278760968653933f};
    return make_float2(c[m], -s[m]);
  }
};
template <> struct Wc<8> {
  static __device__ __forceinline__ float2 w(int m) {
    constexpr float c[8] = {1.f, 0.70710678118654752f, 0.f, -0.70710678118654752f, -1.f,
                            -0.70710678118654752f, 0.f, 0.70710678118654752f};
    constexpr float s[8] = {0.f, 0.70710678118654752f, 1.f, 0.70710678118654752f, 0.f,
                            -0.70710678118654752f, -1.f, -0.70710678118654752f};
    return make_float2(c[m], -s[m]);
  }
};

// Cooley-Tukey composite of size R1 * R2 in registers:
//   input  n = R2 * n1 + n2,  output k = k1 + R1 * k2
template <int R1, int R2>
__device__ __forceinline__ void dft_composite(float2 (&v)[R1 * R2]) {
  constexpr int N = R1 * R2;
  float2 y[R2][R1];
#pragma unroll
  for (int n2 = 0; n2 < R2; ++n2) {
    float2 col[R1];
#pragma unroll
    for (int n1 = 0; n1 < R1; ++n1) col[n1] = v[R2 * n1 + n2];
    dft<R1>(col);
#pragma unroll
    for (int k1 = 0; k1 < R1; ++k1) {
      const int m = (n2 * k1) % N;
      y[n2][k1] = m == 0 ? col[k1] : cmul(col[k1], Wc<N>::w(m));
    }
  }
#pragma unroll
  for (int k1 = 0; k1 < R1; ++k1) {
    float2 row[R2];
#pragma unroll
    for (int n2 = 0; n2 < R2; ++n2) row[n2] = y[n2][k1];
    dft<R2>(row);
#pragma unroll
    for (int k2 = 0; k2 < R2; ++k2) v[k1 + R1 * k2] = row[k2];
  }
}
template <> __device__ __forceinline__ void dft<16>(float2 (&v)[16]) { dft_composite<4, 4>(v); }
template <> __device__ __forceinline__ void dft<9>(float2 (&v)[9]) { dft_composite<3, 3>(v); }
template <> __device__ __forceinline__ void dft<8>(float2 (&v)[8]) { dft_composite<4, 2>(v); }

struct StageInfo {
  int t, ns, step;
  unsigned m_t, m_ns;
};

// One Stockham stage of radix R over `nrows` rows held in `src` (or read from
// global memory when FROM_GLOBAL), writing `dst` (both padded, pitch `pitch`).
// The first stage transforms x - s and records s per row in `shift`.
template <int R, bool FROM_GLOBAL>
__device__ __forceinline__ void stage(const float2* __restrict__ src, float2* __restrict__ dst,
                                      const float2* __restrict__ gsrc, int n2, int pitch,
                                      const float2* __restrict__ tw2, const StageInfo si,
                                      int nrows, float* shift) {
  const int total = nrows * si.t;
  for (int idx = threadIdx.x; idx < total; idx += kSpThreads) {
    const int row = fast_div(idx, si.m_t, si.t);
    const int j = idx - row * si.t;
    float2 v[R];
    const float s = FROM_GLOBAL ? row_shift(gsrc + row * n2) : 0.f;
    if (FROM_GLOBAL && j == 0) shift[row] = s;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      if (FROM_GLOBAL) {
        v[r] = __ldcs(gsrc + row * n2 + j + r * si.t);
        v[r] = make_float2(__fsub_rn(v[r].x, s), __fsub_rn(v[r].y, s));
      } else {
        v[r] = src[row * pitch + pad(j + r * si.t)];
      }
    }
    const int q = fast_div(j, si.m_ns, si.ns);
    const int k = j - q * si.ns;
    if (si.ns > 1) {
      const int base = k * si.step;  // r * k * step < n2
#pragma unroll
      for (int r = 1; r < R; ++r) v[r] = cmul(v[r], tw2[r * base]);
    }
    dft<R>(v);
    const int j0 = q * si.ns * R + k;
#pragma unroll
    for (int r = 0; r < R; ++r) dst[row * pitch + pad(j0 + r * si.ns)] = v[r];
  }
}

template <bool FROM_GLOBAL>
__device__ __forceinline__ void run_stage(int r, const float2* src, float2* dst, const float2* g,
                                          int n2, int pitch, const float2* tw2,
                                          const StageInfo si, int nrows, float* shift) {
  switch (r) {
    case 1: stage<1, FROM_GLOBAL>(src, dst, g, n2, pitch, tw2, si, nrows, shift); break;
    case 2: stage<2, FROM_GLOBAL>(src, dst, g, n2, pitch, tw2, si, nrows, shift); break;
    case 3: stage<3, FROM_GLOBAL>(src, dst, g, n2, pitch, tw2, si, nrows, shift); break;
    case 4: stage<4, FROM_GLOBAL>(src, dst, g, n2, pitch, tw2, si, nrows, shift); break;
    case 5: stage<5, FROM_GLOBAL>(src, dst, g, n2, pitch, tw2, si, nrows, shift); break;
    case 8: stage<8, FROM_GLOBAL>(src, dst, g, n2, pitch, tw2, si, nrows, shift); break;
    case 9: stage<9, FROM_GLOBAL>(src, dst, g, n2, pitch, tw2, si, nrows, shift); break;
    default: stage<16, FROM_GLOBAL>(src, dst, g, n2, pitch, tw2, si, nrows, shift); break;
  }
}

__global__ void __launch_bounds__(kSpThreads) spectrum_kernel(const SpecParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2* buf_a = reinterpret_cast<float2*>(smem_raw);
  float2* buf_b = buf_a + size_t(p.rows_per_block) * p.row_pitch;
  float2* tw2 = buf_b + size_t(p.rows_per_block) * p.row_pitch;
  float2* twn = tw2 + p.n2;
  __shared__ float shift[kSpMaxRows];

  for (int i = threadIdx.x; i < p.n2; i += kSpThreads) tw2[i] = p.tw2[i];
  for (int i = threadIdx.x; i <= p.n2; i += kSpThreads) twn[i] = p.twn[i];
  __syncthreads();

  const int64_t slot = blockIdx.x / p.nblk;
  const int blk = blockIdx.x % p.nblk;
  const int row0 = blk * p.rows_per_block;
  const int nrows = min(p.rows_per_block, p.nrow - row0);
  const int total_out = nrows * p.nk;
  const unsigned m_nk = (unsigned)(((1ull << 32) + p.nk - 1) / p.nk);

  float acc[kSpMaxAcc];
#pragma unroll
  for (int i = 0; i < kSpMaxAcc; ++i) acc[i] = 0.f;

  for (int ti = 0; ti < p.ntimes; ++ti) {
    const int64_t field = int64_t(ti) * p.nfield_out + slot;
    const float2* g =
        reinterpret_cast<const float2*>(p.x + (field * p.nrow + row0) * int64_t(p.n));
    float2* src = buf_b;
    float2* dst = buf_a;
    int ns = 1;
    for (int s = 0; s < p.nstage; ++s) {
      const int r = p.radix[s];
      StageInfo si;
      si.t = p.n2 / r;
      si.ns = ns;
      si.step = p.n2 / (ns * r);
      si.m_t = (unsigned)(((1ull << 32) + si.t - 1) / si.t);
      si.m_ns = (unsigned)(((1ull << 32) + ns - 1) / ns);
      if (s == 0) run_stage<true>(r, src, dst, g, p.n2, p.row_pitch, tw2, si, nrows, shift);
      else run_stage<false>(r, src, dst, g, p.n2, p.row_pitch, tw2, si, nrows, shift);
      __syncthreads();
      float2* tmp = src;
      src = dst;
      dst = tmp;
      ns *= r;
    }
    // `src` now holds Z = DFT_N2(z).  Split into the real-input spectrum:
    //   X_k = (Z_k + conj Z_{N2-k}) / 2 - (i/2) W_N^k (Z_k - conj Z_{N2-k})
#pragma unroll
    for (int it = 0; it < kSpMaxAcc; ++it) {
      const int idx = threadIdx.x + it * kSpThreads;
      if (idx < total_out) {
        const int row = static_cast<int>(__umulhi(static_cast<unsigned>(idx), m_nk));
        const int k = idx - row * p.nk;
        const float2 zk = src[row * p.row_pitch + pad(k == p.n2 ? 0 : k)];
        float2 zc = src[row * p.row_pitch + pad(k == 0 ? 0 : p.n2 - k)];
        zc.y = -zc.y;
        const float2 e = make_float2(0.5f * (zk.x + zc.x), 0.5f * (zk.y + zc.y));
        const float2 d = csub(zk, zc);
        const float2 o = make_float2(0.5f * d.y, -0.5f * d.x);
        float2 xk = cadd(e, cmul(twn[k], o));
        if (k == 0) xk.x += float(p.n) * shift[row];
        const float pw = (xk.x * xk.x + xk.y * xk.y) * (k == 0 ? 1.f : 2.f) * p.scale[row0 + row];
        acc[it] += pw;
      }
    }
    __syncthreads();  // buffers are reused by the next time step
  }

#pragma unroll
  for (int it = 0; it < kSpMaxAcc; ++it) {
    const int idx = threadIdx.x + it * kSpThreads;
    if (idx < total_out) {
      float* o = p.out + (slot * p.nrow + row0) * int64_t(p.nk) + idx;
      *o = p.accumulate ? *o + acc[it] : acc[it];
    }
  }
}

// ---------------------------------------------------------------------------
// Fixed-plan variant: N2 and the (up to three) radices are template constants,
// so every division, stride, twiddle step and padded index folds at compile
// time, and the post-pass handles the bins k and N2 - k together (they share
// both loads and the complex product W_N^k * O):
//     X_k = E + W O,   X_{N2-k} = conj(E - W O).
// ---------------------------------------------------------------------------
// The first stage (FROM_GLOBAL) transforms x - s and records s per row in `shift`.
template <int R, int NS, int N2, bool FROM_GLOBAL>
__device__ __forceinline__ void stage_ct(const float2* __restrict__ src, float2* __restrict__ dst,
                                         const float2* __restrict__ gsrc,
                                         const float2* __restrict__ tw2, int nrows,
                                         float* shift) {
  constexpr int T = N2 / R;
  constexpr int STEP = N2 / (NS * R);
  constexpr int PITCH = N2 + (N2 >> 4) + 1;
  const int total = nrows * T;
  for (int idx = threadIdx.x; idx < total; idx += kSpThreads) {
    const int row = idx / T;
    const int j = idx - row * T;
    float2 v[R];
    const float s = FROM_GLOBAL ? row_shift(gsrc + row * N2) : 0.f;
    if (FROM_GLOBAL && j == 0) shift[row] = s;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      if (FROM_GLOBAL) {
        v[r] = __ldcs(gsrc + row * N2 + j + r * T);
        v[r] = make_float2(__fsub_rn(v[r].x, s), __fsub_rn(v[r].y, s));
      } else {
        v[r] = src[row * PITCH + pad(j + r * T)];
      }
    }
    const int q = j / NS;
    const int k = j - q * NS;
    if (NS > 1) {
      const int base = k * STEP;
#pragma unroll
      for (int r = 1; r < R; ++r) v[r] = cmul(v[r], tw2[r * base]);
    }
    dft<R>(v);
    const int j0 = q * (NS * R) + k;
#pragma unroll
    for (int r = 0; r < R; ++r) dst[row * PITCH + pad(j0 + r * NS)] = v[r];
  }
}

template <int N2, int R0, int R1, int R2>
__global__ void __launch_bounds__(kSpThreads) spectrum_fixed_kernel(const SpecParams p) {
  static_assert(R0 * R1 * R2 == N2, "radix plan must multiply to N2");
  constexpr int PITCH = N2 + (N2 >> 4) + 1;
  constexpr int NK = N2 + 1;
  constexpr int NPAIR = N2 / 2 + 1;  // pair p handles bins p and N2 - p
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2* buf_a = reinterpret_cast<float2*>(smem_raw);
  float2* buf_b = buf_a + size_t(p.rows_per_block) * PITCH;
  float2* tw2 = buf_b + size_t(p.rows_per_block) * PITCH;
  float2* twn = tw2 + N2;
  __shared__ float shift[kSpMaxRows];  // per row of the block: the first stage's shift

  for (int i = threadIdx.x; i < N2; i += kSpThreads) tw2[i] = p.tw2[i];
  for (int i = threadIdx.x; i <= N2; i += kSpThreads) twn[i] = p.twn[i];
  __syncthreads();

  const int64_t slot = blockIdx.x / p.nblk;
  const int blk = blockIdx.x % p.nblk;
  const int row0 = blk * p.rows_per_block;
  const int nrows = min(p.rows_per_block, p.nrow - row0);
  const int total_pairs = nrows * NPAIR;

  constexpr int kPairIters = kSpMaxAcc / 2;
  float acc_lo[kPairIters], acc_hi[kPairIters];
  float acc_dc = 0.f, acc_ny = 0.f;  // bins 0 and N2 of row threadIdx.x
#pragma unroll
  for (int i = 0; i < kPairIters; ++i) { acc_lo[i] = 0.f; acc_hi[i] = 0.f; }

  for (int ti = 0; ti < p.ntimes; ++ti) {
    const int64_t field = int64_t(ti) * p.nfield_out + slot;
    const float2* g =
        reinterpret_cast<const float2*>(p.x + (field * p.nrow + row0) * int64_t(2 * N2));
    stage_ct<R0, 1, N2, true>(nullptr, buf_a, g, tw2, nrows, shift);
    __syncthreads();
    const float2* z = buf_a;
    if (R1 > 1) {
      stage_ct<R1, R0, N2, false>(buf_a, buf_b, g, tw2, nrows, shift);
      __syncthreads();
      z = buf_b;
      if (R2 > 1) {
        stage_ct<R2, R0 * R1, N2, false>(buf_b, buf_a, g, tw2, nrows, shift);
        __syncthreads();
        z = buf_a;
      }
    }
#pragma unroll
    for (int it = 0; it < kPairIters; ++it) {
      const int idx = threadIdx.x + it * kSpThreads;
      const int row = idx / NPAIR;
      const int k = idx - row * NPAIR;
      if (idx < total_pairs && k != 0) {
        const float2 zk = z[row * PITCH + pad(k)];
        float2 zc = z[row * PITCH + pad(k == 0 ? 0 : N2 - k)];
        zc.y = -zc.y;
        const float2 e = make_float2(0.5f * (zk.x + zc.x), 0.5f * (zk.y + zc.y));
        const float2 d = csub(zk, zc);
        const float2 o = make_float2(0.5f * d.y, -0.5f * d.x);
        const float2 wo = cmul(twn[k], o);
        const float2 xa = cadd(e, wo), xb = csub(e, wo);
        const float sc = p.scale[row0 + row];
        acc_lo[it] += (xa.x * xa.x + xa.y * xa.y) * (k == 0 ? 1.f : 2.f) * sc;
        acc_hi[it] += (xb.x * xb.x + xb.y * xb.y) * 2.f * sc;
      }
    }
    // bins 0 and N2 of row threadIdx.x: X_0 = Re Z_0 + Im Z_0 + N s (the shift
    // back), X_N2 = Re Z_0 - Im Z_0 (the shift cancels)
    if (threadIdx.x < nrows) {
      const int row = threadIdx.x;
      const float2 z0 = z[row * PITCH];
      const float x0 = (z0.x + z0.y) + float(2 * N2) * shift[row], xn = z0.x - z0.y;
      const float sc = p.scale[row0 + row];
      acc_dc += x0 * x0 * sc;
      acc_ny += xn * xn * 2.f * sc;
    }
    __syncthreads();  // buffers are reused by the next time step
  }

#pragma unroll
  for (int it = 0; it < kPairIters; ++it) {
    const int idx = threadIdx.x + it * kSpThreads;
    const int row = idx / NPAIR;
    const int k = idx - row * NPAIR;
    if (idx < total_pairs && k != 0) {
      float* o = p.out + ((slot * p.nrow + row0 + row) * int64_t(NK));
      o[k] = p.accumulate ? o[k] + acc_lo[it] : acc_lo[it];
      if (2 * k != N2) o[N2 - k] = p.accumulate ? o[N2 - k] + acc_hi[it] : acc_hi[it];
    }
  }
  if (threadIdx.x < nrows) {
    float* o = p.out + ((slot * p.nrow + row0 + threadIdx.x) * int64_t(NK));
    o[0] = p.accumulate ? o[0] + acc_dc : acc_dc;
    o[N2] = p.accumulate ? o[N2] + acc_ny : acc_ny;
  }
}

template <int N2, int R0, int R1, int R2>
static int launch_fixed(wb2_ctx* ctx, const SpecParams& p, size_t smem, unsigned grid) {
  auto kernel = spectrum_fixed_kernel<N2, R0, R1, R2>;
  if (smem + kSpStaticSmem > 48 * 1024)
    WB2_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      static_cast<int>(smem)));
  kernel<<<grid, kSpThreads, smem, ctx->stream>>>(p);
  WB2_CUDA_TRY(cudaGetLastError());
  return WB2_OK;
}

// Returns 1 if a fixed-plan kernel exists for n2 (and was launched), else 0.
static int try_fixed(wb2_ctx* ctx, const SpecParams& p, size_t smem, unsigned grid) {
  const char* force = getenv("WB2_SPECTRUM_PATH");
  if (force && strcmp(force, "generic") == 0) return 0;
  if (p.rows_per_block * (p.n2 / 2 + 1) > (kSpMaxAcc / 2) * kSpThreads) return 0;
  int rc;
  switch (p.n2) {
    case 720: rc = launch_fixed<720, 16, 9, 5>(ctx, p, smem, grid); break;  // 1440 (0.25 deg)
    case 360: rc = launch_fixed<360, 9, 8, 5>(ctx, p, smem, grid); break;   // 720  (0.5 deg)
    case 180: rc = launch_fixed<180, 9, 5, 4>(ctx, p, smem, grid); break;   // 360  (1 deg)
    case 120: rc = launch_fixed<120, 8, 5, 3>(ctx, p, smem, grid); break;   // 240  (1.5 deg)
    case 256: rc = launch_fixed<256, 16, 16, 1>(ctx, p, smem, grid); break; // 512
    case 32: rc = launch_fixed<32, 16, 2, 1>(ctx, p, smem, grid); break;    // 64   (5.625 deg)
    default: return 0;
  }
  return rc == WB2_OK ? 1 : rc;
}

static bool factorize(int n2, int* radix, int* nstage) {
  int n = n2, ns = 0;
  const int order[7] = {16, 9, 8, 5, 4, 3, 2};
  for (int oi = 0; oi < 7; ++oi) {
    const int r = order[oi];
    while (n % r == 0) {
      if (ns >= kSpMaxStages) return false;
      radix[ns++] = r;
      n /= r;
    }
  }
  if (n != 1) return false;
  if (ns == 0) radix[ns++] = 1;
  *nstage = ns;
  return true;
}

// spectrum_pfa.cu: prime-factor / row-pair / TMA kernel for 1440, 720 and 240
// longitudes (1 = handled, 0 = not eligible, < 0 = error)
int spectrum_pfa_try(wb2_ctx* ctx, const float* x, int64_t nfield, int32_t nrow, int32_t ncol,
                     const double* scale, float* out, int mode, int64_t nslot);

// out[slot][k] = sum_row spec[slot][row][k]   (rows already carry their weights;
// rows of zero weight are skipped, so that a NaN or inf outside a latitude band
// does not reach the band's sum as 0 * NaN)
__global__ void latsum_rows_kernel(const float* __restrict__ spec,
                                   const unsigned char* __restrict__ keep,
                                   float* __restrict__ out, int64_t nslot, int nrow, int nk,
                                   int accumulate) {
  const int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
  if (i >= nslot * nk) return;
  const int64_t slot = i / nk;
  const int k = static_cast<int>(i - slot * nk);
  float s = 0.f;
  for (int r = 0; r < nrow; ++r)
    if (keep[r]) s += spec[(slot * nrow + r) * int64_t(nk) + k];
  out[i] = accumulate ? out[i] + s : s;
}

// wb2_zonal_spectrum_latsum; accumulate != 0 adds to `out` (the host-streaming
// entry sums groups of time steps this way).
int spectrum_latsum_impl(wb2_ctx* ctx, const float* x, int64_t nfield, int32_t nrow,
                         int32_t ncol, const double* scale, float* out, int64_t nfield_out,
                         int accumulate) {
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_REQUIRE(nrow > 0 && ncol > 1, "bad grid %d x %d", nrow, ncol);
  WB2_REQUIRE(nfield >= 0, "nfield < 0");
  if (nfield == 0) return WB2_OK;
  WB2_REQUIRE(x && out && scale, "NULL argument");
  WB2_REQUIRE(nfield_out > 0 && nfield % nfield_out == 0,
              "nfield (%lld) must be a multiple of nfield_out (%lld)",
              static_cast<long long>(nfield), static_cast<long long>(nfield_out));
  DeviceGuard guard(ctx->device);
  const int prc = spectrum_pfa_try(ctx, x, nfield, nrow, ncol, scale, out, accumulate ? 3 : 2,
                                   nfield_out);
  if (prc != 0) return prc < 0 ? prc : WB2_OK;
  // other row lengths / unaligned data: per-row spectra (time-summed) into
  // scratch, then the row sum
  const int nk = ncol / 2 + 1;
  const size_t need = size_t(nfield_out) * nrow * nk * sizeof(float);
  WB2_TRY(grow_buffer(ctx, ctx->scratch, ctx->scratch_cap, need));
  float* spec = static_cast<float*>(ctx->scratch);
  WB2_CUDA_TRY(cudaMemsetAsync(spec, 0, need, ctx->stream));
  WB2_TRY(wb2_zonal_spectrum(ctx, x, nfield, nrow, ncol, scale, spec, 1, nfield_out));
  std::vector<unsigned char> keep(nrow);
  for (int r = 0; r < nrow; ++r) keep[r] = scale[r] != 0.0;
  Packer pk(ctx);
  const size_t ok = pk.add(keep.data(), keep.size());
  WB2_TRY(pk.commit());
  const int64_t n = nfield_out * nk;
  latsum_rows_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, ctx->stream>>>(
      spec, pk.dev<unsigned char>(ok), out, nfield_out, nrow, nk, accumulate);
  WB2_CUDA_TRY(cudaGetLastError());
  ctx->launches += 1;
  WB2_TRY(pk.release());
  return WB2_OK;
}

}  // namespace wb2

using namespace wb2;

extern "C" int wb2_zonal_spectrum_latsum(wb2_ctx* ctx, const float* x, int64_t nfield,
                                         int32_t nrow, int32_t ncol, const double* scale,
                                         float* out, int64_t nfield_out) {
  WB2_NVTX("wb2_zonal_spectrum_latsum");
  return spectrum_latsum_impl(ctx, x, nfield, nrow, ncol, scale, out, nfield_out, 0);
}

extern "C" int wb2_zonal_spectrum(wb2_ctx* ctx, const float* x, int64_t nfield, int32_t nrow,
                                  int32_t ncol, const double* scale, float* out,
                                  int32_t accumulate, int64_t nfield_out) {
  WB2_NVTX("wb2_zonal_spectrum");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_REQUIRE(nrow > 0 && ncol > 1, "bad grid %d x %d", nrow, ncol);
  WB2_REQUIRE(nfield >= 0, "nfield < 0");
  if (nfield == 0) return WB2_OK;
  WB2_REQUIRE(x && out && scale, "NULL argument");
  if (!accumulate) nfield_out = nfield;
  WB2_REQUIRE(nfield_out > 0 && nfield % nfield_out == 0,
              "nfield (%lld) must be a multiple of nfield_out (%lld)",
              static_cast<long long>(nfield), static_cast<long long>(nfield_out));
  // the Stockham kernels read each row as float2
  WB2_REQUIRE((reinterpret_cast<uintptr_t>(x) & 7) == 0, "wb2_zonal_spectrum: x must be 8-byte aligned");
  if (ncol % 2 != 0) {
    set_error("wb2_zonal_spectrum: odd number of longitudes (%d) is not supported", ncol);
    return WB2_EUNSUPPORTED;
  }
  SpecParams p;
  p.n = ncol; p.n2 = ncol / 2; p.nk = p.n2 + 1; p.nrow = nrow;
  if (p.n2 == 1) {
    p.nstage = 1;
    p.radix[0] = 1;
  } else if (!factorize(p.n2, p.radix, &p.nstage)) {
    set_error("wb2_zonal_spectrum: %d longitudes: N/2 must factor into 2, 3 and 5", ncol);
    return WB2_EUNSUPPORTED;
  }
  DeviceGuard guard(ctx->device);
  {
    const int prc = spectrum_pfa_try(ctx, x, nfield, nrow, ncol, scale, out,
                                     accumulate ? 1 : 0, nfield_out);
    if (prc != 0) return prc < 0 ? prc : WB2_OK;
    const char* force = getenv("WB2_SPECTRUM_PATH");
    if (force && strcmp(force, "pfa") == 0) {  // tests: fail instead of falling back
      set_error("wb2_zonal_spectrum: WB2_SPECTRUM_PATH=pfa but %d longitudes / this "
                "alignment are not eligible for the prime-factor kernel", ncol);
      return WB2_EUNSUPPORTED;
    }
  }

  // host tables in double precision, rounded once to float32
  std::vector<float2> tw2(p.n2), twn(p.n2 + 1);
  const double two_pi = 6.283185307179586476925286766559;
  for (int k = 0; k < p.n2; ++k) {
    const double a = -two_pi * k / p.n2;
    tw2[k] = make_float2(static_cast<float>(cos(a)), static_cast<float>(sin(a)));
  }
  for (int k = 0; k <= p.n2; ++k) {
    const double a = -two_pi * k / p.n;
    twn[k] = make_float2(static_cast<float>(cos(a)), static_cast<float>(sin(a)));
  }
  std::vector<float> sc(nrow);
  for (int i = 0; i < nrow; ++i)
    sc[i] = static_cast<float>(scale[i] / (double(ncol) * double(ncol)));

  // rows per CTA: ~46 KB per ping-pong buffer, bounded by the register
  // accumulators (kSpMaxAcc outputs per thread) and by fast_div's range
  p.row_pitch = p.n2 + (p.n2 >> 4) + 1;
  int rpb = static_cast<int>((46 * 1024) / (size_t(p.row_pitch) * sizeof(float2)));
  if (rpb < 1) rpb = 1;
  if (rpb > kSpMaxRows) rpb = kSpMaxRows;
  while (rpb > 1 && rpb * p.nk > kSpMaxAcc * kSpThreads) --rpb;
  WB2_REQUIRE(rpb * p.nk <= kSpMaxAcc * kSpThreads && rpb * p.nk < (1 << 20),
              "wb2_zonal_spectrum: %d longitudes exceed the supported row length", ncol);
  if (rpb > nrow) rpb = nrow;
  p.rows_per_block = rpb;
  p.nblk = (nrow + rpb - 1) / rpb;
  p.nfield_out = nfield_out;
  p.ntimes = static_cast<int>(nfield / nfield_out);
  p.accumulate = accumulate ? 1 : 0;
  const size_t smem = (size_t(2) * rpb * p.row_pitch + p.n2 + p.n2 + 1) * sizeof(float2);
  WB2_REQUIRE(smem <= 220 * 1024, "wb2_zonal_spectrum: row too long for shared memory");
  (void)magic;

  Packer pk(ctx);
  size_t o1 = pk.add(tw2.data(), tw2.size() * sizeof(float2));
  size_t o2 = pk.add(twn.data(), twn.size() * sizeof(float2));
  size_t o3 = pk.add(sc.data(), sc.size() * sizeof(float));
  WB2_TRY(pk.commit());
  p.x = x; p.out = out;
  p.tw2 = pk.dev<float2>(o1); p.twn = pk.dev<float2>(o2); p.scale = pk.dev<float>(o3);
  const unsigned grid = static_cast<unsigned>(nfield_out * p.nblk);
  const int frc = try_fixed(ctx, p, smem, grid);
  if (frc < 0) return frc;
  if (frc == 0) {
    if (smem + kSpStaticSmem > 48 * 1024)
      WB2_CUDA_TRY(cudaFuncSetAttribute(spectrum_kernel,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        static_cast<int>(smem)));
    spectrum_kernel<<<grid, kSpThreads, smem, ctx->stream>>>(p);
    WB2_CUDA_TRY(cudaGetLastError());
  }
  ctx->launches += 1;
  WB2_TRY(pk.release());
  return WB2_OK;
}

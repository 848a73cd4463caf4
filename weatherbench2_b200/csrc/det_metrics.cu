// K1 -- fused deterministic metrics (sm_90a).
//
// One pass over forecast / truth / climatology slabs produces, for every field
// and every region, the six weighted sums behind MSE, RMSE, MAE, Bias and ACC
// plus the matching sums of weights (xarray's `sum_of_weights`):
//   weatherbench2/metrics.py:141-163 (_spatial_average), :283-301 (MSE),
//   :251-269 (RMSE), :323-330 (MAE), :352-359 (Bias), :387-414 (ACC),
//   :189-202 (WindVectorMSE).
// The reference re-reads the chunk once per metric x region
// (weatherbench2/evaluation.py:408-435); here the chunk is read exactly once.
//
// Roofline: HBM-bound streaming reduce, 12 B per cell (f, t, c in f32), ~0 B
// written.  No tensor cores (there is no contraction).
//
// Work decomposition.  grid = fields x row blocks; a CTA of 8 warps owns
// `rows_per_block` consecutive rows of one field, warp w takes rows w, w+8, ...
// A row is split into the column segments the regions induce (usually one);
// within a (row, segment) every cell has the same separable region weight, so
// lanes accumulate UNWEIGHTED f32 partial sums over 128-bit streaming loads,
// one butterfly reduces them, and lane r applies region r's float64 weight
// row_w[r][row] * seg_w[r][seg] to its own float64 accumulators.  CTAs write
// float64 partials; a second tiny kernel adds them in a fixed order
// (deterministic, no float atomics).
#include "region_reduce.cuh"

namespace wb2 {

constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
constexpr int kUnroll = 4;

struct DetParams {
  const void* f;
  const void* t;
  const void* c;
  const void* g;  // 4th operand (wind-vector mode: fu, tu, fv, tv = f, t, c, g)
  const int64_t* off_f;
  const int64_t* off_t;
  const int64_t* off_c;
  const int64_t* off_g;
  const double* row_w;       // [R][nrow]
  const int32_t* seg_start;  // [nseg + 1]
  const double* seg_w;       // [R][nseg]
  const float* col_w;        // [ncol] or null
  const float* cell_w;       // [nrow][ncol] or null
  double* partial;           // [nfield][nblk][R][WB2_DET_NSTAT]
  int32_t nrow, ncol;
  int64_t row_stride;
  int32_t nregion, nseg;
  int32_t zero_skip;
  int32_t rows_per_block;
  int32_t nblk;
};

enum { MODE_PLAIN = 0, MODE_CLIM = 1, MODE_VECTOR = 2 };

template <int MODE> struct ModeTraits;
template <> struct ModeTraits<MODE_PLAIN> { static constexpr int NSUM = 3, NOPER = 2; };
template <> struct ModeTraits<MODE_CLIM> { static constexpr int NSUM = 6, NOPER = 3; };
template <> struct ModeTraits<MODE_VECTOR> { static constexpr int NSUM = 1, NOPER = 4; };

template <int MODE, bool SKIPNA>
struct Counts {
  static constexpr int NCNT = SKIPNA ? (MODE == MODE_CLIM ? 4 : 1) : 1;
};

template <typename A>
__device__ __forceinline__ bool is_nan(A v) { return v != v; }

// Accumulate one cell.  `wc` is the non-separable part of the weight
// (col_w * cell_w); WEIGHTED == false means wc == 1.
template <typename A, int MODE, bool SKIPNA, bool WEIGHTED>
__device__ __forceinline__ void accumulate_cell(A f, A t, A c, A g, A wc,
                                                bool zero_skip, A* acc) {
  constexpr int NSUM = ModeTraits<MODE>::NSUM;
  if (WEIGHTED) {
    // metrics.py:160  `dataset.where(weights > 0, 0)`: a zero-weight cell
    // contributes nothing, whatever it holds.
    if (zero_skip && wc == A(0)) return;
  }
  if (MODE == MODE_VECTOR) {
    A du = f - t, dv = c - g;
    A v0 = du * du + dv * dv;  // metrics.py:198
    if (SKIPNA) {
      bool ok = !is_nan(v0);
      A w = ok ? wc : A(0);
      acc[0] += ok ? (WEIGHTED ? wc * v0 : v0) : A(0);
      acc[NSUM] += WEIGHTED ? w : (ok ? A(1) : A(0));
    } else {
      acc[0] += WEIGHTED ? wc * v0 : v0;
      acc[NSUM] += WEIGHTED ? wc : A(1);
    }
    return;
  }
  A d = f - t;
  A v0 = d * d, v1 = fabs(d), v2 = d;
  if (SKIPNA) {
    bool ok = !is_nan(d);
    if (ok) {
      acc[0] += WEIGHTED ? wc * v0 : v0;
      acc[1] += WEIGHTED ? wc * v1 : v1;
      acc[2] += WEIGHTED ? wc * v2 : v2;
      acc[NSUM] += WEIGHTED ? wc : A(1);
    }
  } else {
    acc[0] += WEIGHTED ? wc * v0 : v0;
    acc[1] += WEIGHTED ? wc * v1 : v1;
    acc[2] += WEIGHTED ? wc * v2 : v2;
    acc[NSUM] += WEIGHTED ? wc : A(1);
  }
  if (MODE == MODE_CLIM) {
    A fa = f - c, ta = t - c;  // metrics.py:405-406
    A v3 = fa * ta, v4 = fa * fa, v5 = ta * ta;
    if (SKIPNA) {
      if (!is_nan(v3)) { acc[3] += WEIGHTED ? wc * v3 : v3; acc[NSUM + 1] += WEIGHTED ? wc : A(1); }
      if (!is_nan(fa)) { acc[4] += WEIGHTED ? wc * v4 : v4; acc[NSUM + 2] += WEIGHTED ? wc : A(1); }
      if (!is_nan(ta)) { acc[5] += WEIGHTED ? wc * v5 : v5; acc[NSUM + 3] += WEIGHTED ? wc : A(1); }
    } else {
      acc[3] += WEIGHTED ? wc * v3 : v3;
      acc[4] += WEIGHTED ? wc * v4 : v4;
      acc[5] += WEIGHTED ? wc * v5 : v5;
    }
  }
}

template <typename T, int VEC> struct VecType;
template <> struct VecType<float, 4> { using type = float4; };
template <> struct VecType<float, 1> { using type = float; };
template <> struct VecType<double, 2> { using type = double2; };
template <> struct VecType<double, 1> { using type = double; };

template <typename T, int VEC>
struct Pack {
  T v[VEC];
};

template <typename T, int VEC>
__device__ __forceinline__ Pack<T, VEC> load_pack(const T* p) {
  using V = typename VecType<T, VEC>::type;
  V raw = ldg_stream(reinterpret_cast<const V*>(p));
  Pack<T, VEC> r;
  memcpy(r.v, &raw, sizeof(V));
  return r;
}

template <int VEC>
__device__ __forceinline__ Pack<float, VEC> load_weights(const float* p) {
  Pack<float, VEC> r;
#pragma unroll
  for (int i = 0; i < VEC; ++i) r.v[i] = p[i];
  return r;
}

template <typename T, int VEC, int MODE, bool SKIPNA, bool WEIGHTED>
__global__ void __launch_bounds__(kThreads)
det_metrics_kernel(const DetParams p) {
  constexpr int NSUM = ModeTraits<MODE>::NSUM;
  constexpr int NOPER = ModeTraits<MODE>::NOPER;
  constexpr int NCNT = Counts<MODE, SKIPNA>::NCNT;
  constexpr int NS = NSUM + NCNT;
  using A = T;  // lane accumulator type follows the data type

  extern __shared__ __align__(16) unsigned char smem_raw[];
  double* red = reinterpret_cast<double*>(smem_raw);           // [kWarps][32][NS]
  float* s_colw = reinterpret_cast<float*>(red + kWarps * 32 * NS);  // [ncol]

  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int64_t field = blockIdx.x / p.nblk;
  const int blk = blockIdx.x % p.nblk;
  const int R = p.nregion;

  if (WEIGHTED && p.col_w) {
    for (int i = threadIdx.x; i < p.ncol; i += kThreads) s_colw[i] = p.col_w[i];
    __syncthreads();
  }

  const T* __restrict__ pf = static_cast<const T*>(p.f) + p.off_f[field];
  const T* __restrict__ pt = static_cast<const T*>(p.t) + p.off_t[field];
  const T* __restrict__ pc = NOPER >= 3 ? static_cast<const T*>(p.c) + p.off_c[field] : nullptr;
  const T* __restrict__ pg = NOPER >= 4 ? static_cast<const T*>(p.g) + p.off_g[field] : nullptr;

  double accd[NS];
#pragma unroll
  for (int i = 0; i < NS; ++i) accd[i] = 0.0;

  const int row0 = blk * p.rows_per_block;
  const int row1 = min(p.nrow, row0 + p.rows_per_block);
  const bool zero_skip = p.zero_skip != 0;

  for (int row = row0 + warp; row < row1; row += kWarps) {
    const int64_t rbase = int64_t(row) * p.row_stride;
    for (int k = 0; k < p.nseg; ++k) {
      const int s = p.seg_start[k];
      const int e = p.seg_start[k + 1];
      A acc[NS];
#pragma unroll
      for (int i = 0; i < NS; ++i) acc[i] = A(0);

      // Segment boundaries need not be VEC-aligned: peel up to VEC-1 head and
      // tail cells (one lane each, scalar loads), vector body in between.
      int s_al = s, e_al = e;
      if (VEC > 1) {
        s_al = min(e, (s + VEC - 1) / VEC * VEC);
        e_al = max(s_al, e / VEC * VEC);
        const int nh = s_al - s, nt = e - e_al;
        if (lane < nh + nt) {
          const int col = lane < nh ? s + lane : e_al + (lane - nh);
          A wc = A(1);
          if (WEIGHTED) {
            if (p.col_w) wc *= A(s_colw[col]);
            if (p.cell_w) wc *= A(p.cell_w[int64_t(row) * p.ncol + col]);
          }
          accumulate_cell<A, MODE, SKIPNA, WEIGHTED>(
              ldg_stream(pf + rbase + col), ldg_stream(pt + rbase + col),
              NOPER >= 3 ? ldg_stream(pc + rbase + col) : A(0),
              NOPER >= 4 ? ldg_stream(pg + rbase + col) : A(0), wc, zero_skip, acc);
        }
      }
      // lanes stride over VEC-wide packs; kUnroll packs are loaded before use
      for (int c0 = s_al + lane * VEC; c0 < e_al; c0 += 32 * VEC * kUnroll) {
        Pack<T, VEC> xf[kUnroll], xt[kUnroll], xc[kUnroll], xg[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
          const int col = c0 + u * 32 * VEC;
          if (col < e_al) {
            xf[u] = load_pack<T, VEC>(pf + rbase + col);
            xt[u] = load_pack<T, VEC>(pt + rbase + col);
            if (NOPER >= 3) xc[u] = load_pack<T, VEC>(pc + rbase + col);
            if (NOPER >= 4) xg[u] = load_pack<T, VEC>(pg + rbase + col);
          }
        }
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
          const int col = c0 + u * 32 * VEC;
          if (col < e_al) {
            Pack<float, VEC> wcol, wcell;
            if (WEIGHTED) {
              if (p.col_w) wcol = load_weights<VEC>(s_colw + col);
              if (p.cell_w) wcell = load_weights<VEC>(p.cell_w + int64_t(row) * p.ncol + col);
            }
#pragma unroll
            for (int v = 0; v < VEC; ++v) {
              A wc = A(1);
              if (WEIGHTED) {
                if (p.col_w) wc *= A(wcol.v[v]);
                if (p.cell_w) wc *= A(wcell.v[v]);
              }
              accumulate_cell<A, MODE, SKIPNA, WEIGHTED>(
                  xf[u].v[v], xt[u].v[v], NOPER >= 3 ? xc[u].v[v] : A(0),
                  NOPER >= 4 ? xg[u].v[v] : A(0), wc, zero_skip, acc);
            }
          }
        }
      }

      // (row, segment) totals -> every lane; lane r applies region r's weight
#pragma unroll
      for (int i = 0; i < NS; ++i) acc[i] = warp_sum(acc[i]);
      if (lane < R) {
        const double w = p.row_w[int64_t(lane) * p.nrow + row] *
                         p.seg_w[lane * p.nseg + k];
        if (!(zero_skip && w == 0.0)) {
#pragma unroll
          for (int i = 0; i < NS; ++i) accd[i] += w * double(acc[i]);
        }
      }
    }
  }

  // CTA combine (fixed order) and write the partial in the public stat layout
#pragma unroll
  for (int i = 0; i < NS; ++i) red[(warp * 32 + lane) * NS + i] = accd[i];
  __syncthreads();
  double* out = p.partial + (field * p.nblk + blk) * int64_t(R) * WB2_DET_NSTAT;
  for (int idx = threadIdx.x; idx < R * WB2_DET_NSTAT; idx += kThreads) {
    const int r = idx / WB2_DET_NSTAT;
    const int st = idx % WB2_DET_NSTAT;
    const int slot = k1_slot(st, NSUM, MODE == MODE_CLIM, SKIPNA);
    double v = 0.0;
    if (slot >= 0) {
#pragma unroll
      for (int w = 0; w < kWarps; ++w) v += red[(w * 32 + r) * NS + slot];
    }
    out[idx] = v;
  }
}

template <typename T, int VEC, int MODE>
static int launch_mode(wb2_ctx* ctx, const DetParams& p, int64_t nfield, bool skipna,
                       bool weighted) {
  constexpr int NSUM = ModeTraits<MODE>::NSUM;
  const int ns = NSUM + (skipna ? Counts<MODE, true>::NCNT : Counts<MODE, false>::NCNT);
  size_t smem = size_t(kWarps) * 32 * ns * sizeof(double) +
                (weighted && p.col_w ? size_t(p.ncol) * sizeof(float) : 0);
  const dim3 grid(static_cast<unsigned>(nfield * p.nblk));
  auto go = [&](auto kernel) { return launch_kernel(ctx, kernel, grid, kThreads, smem, p); };
  if (skipna) {
    if (weighted) return go(det_metrics_kernel<T, VEC, MODE, true, true>);
    return go(det_metrics_kernel<T, VEC, MODE, true, false>);
  }
  if (weighted) return go(det_metrics_kernel<T, VEC, MODE, false, true>);
  return go(det_metrics_kernel<T, VEC, MODE, false, false>);
}

template <typename T>
static int launch_dtype(wb2_ctx* ctx, const DetParams& p, int64_t nfield, int mode,
                        bool skipna, bool weighted, bool vec_ok) {
  constexpr int VEC = sizeof(T) == 4 ? 4 : 2;
  if (vec_ok) {
    switch (mode) {
      case MODE_PLAIN: return launch_mode<T, VEC, MODE_PLAIN>(ctx, p, nfield, skipna, weighted);
      case MODE_CLIM: return launch_mode<T, VEC, MODE_CLIM>(ctx, p, nfield, skipna, weighted);
      default: return launch_mode<T, VEC, MODE_VECTOR>(ctx, p, nfield, skipna, weighted);
    }
  }
  switch (mode) {
    case MODE_PLAIN: return launch_mode<T, 1, MODE_PLAIN>(ctx, p, nfield, skipna, weighted);
    case MODE_CLIM: return launch_mode<T, 1, MODE_CLIM>(ctx, p, nfield, skipna, weighted);
    default: return launch_mode<T, 1, MODE_VECTOR>(ctx, p, nfield, skipna, weighted);
  }
}

// det_tma.cu: 1 if the kernel ran, 0 if the launch is not eligible, < 0 on error
int det_metrics_tma(wb2_ctx* ctx, bool clim, const void* f, const void* t, const void* c,
                    int64_t nfield, const int64_t* d_off_f, const int64_t* d_off_t,
                    const int64_t* d_off_c, const double* d_row_w, const double* d_seg_w,
                    const wb2_weights* w, int skipna, double* out);

int det_metrics_tma_seg(wb2_ctx* ctx, bool clim, const void* f, const void* t, const void* c,
                        int64_t nfield, const int64_t* d_off_f, const int64_t* d_off_t,
                        const int64_t* d_off_c, const wb2_weights* w, int skipna, double* out);

static bool all_multiple(const int64_t* v, int64_t n, int64_t m) {
  if (!v) return true;
  for (int64_t i = 0; i < n; ++i)
    if (v[i] % m) return false;
  return true;
}

// Shared implementation of wb2_det_metrics / wb2_det_metrics_vector.
int det_metrics_impl(wb2_ctx* ctx, int mode, const void* f, const void* t, const void* c,
                     const void* g, int dtype, int64_t nfield, const int64_t* off_f,
                     const int64_t* off_t, const int64_t* off_c, const int64_t* off_g,
                     const wb2_weights* w, int skipna, double* out) {
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_REQUIRE(dtype == WB2_F32 || dtype == WB2_F64, "dtype must be WB2_F32 or WB2_F64");
  WB2_REQUIRE(nfield >= 0 && nfield <= (int64_t(1) << 24), "nfield out of range: %lld",
              static_cast<long long>(nfield));
  WB2_TRY(validate_weights(w));
  WB2_REQUIRE(out != nullptr, "out is NULL");
  if (nfield == 0) return WB2_OK;
  WB2_REQUIRE(f && t && off_f && off_t, "f/t and their offset tables must not be NULL");
  if (mode == MODE_CLIM) WB2_REQUIRE(c && off_c, "climatology pointer/offsets are NULL");
  if (mode == MODE_VECTOR)
    WB2_REQUIRE(c && g && off_c && off_g, "vector mode needs four operands");
  DeviceGuard guard(ctx->device);

  const size_t esize = dtype == WB2_F32 ? 4 : 8;
  const int vec = dtype == WB2_F32 ? 4 : 2;
  auto aligned16 = [](const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; };
  bool vec_ok = aligned16(f) && aligned16(t) && (!c || aligned16(c)) && (!g || aligned16(g)) &&
                (w->row_stride % vec == 0) && all_multiple(off_f, nfield, vec) &&
                all_multiple(off_t, nfield, vec) &&
                (mode == MODE_PLAIN || all_multiple(off_c, nfield, vec)) &&
                (mode != MODE_VECTOR || all_multiple(off_g, nfield, vec));
  (void)esize;

  // rows per CTA: 4 rows per warp keeps the per-CTA epilogue negligible and
  // gives >= 20 waves on the headline shape (780 fields x 23 blocks).
  const BlockRows br = block_rows(w->nrow, nfield, 4 * kWarps, kWarps, 2 * ctx->num_sms);
  const size_t per_field = size_t(w->nregion) * WB2_DET_NSTAT;
  Packer pk(ctx);
  size_t o_f = pk.add(off_f, nfield * sizeof(int64_t));
  size_t o_t = pk.add(off_t, nfield * sizeof(int64_t));
  size_t o_c = off_c ? pk.add(off_c, nfield * sizeof(int64_t)) : 0;
  size_t o_g = off_g ? pk.add(off_g, nfield * sizeof(int64_t)) : 0;
  const WeightUpload wu(pk, w);
  size_t o_part = pk.reserve(size_t(nfield) * br.nblk * per_field * sizeof(double));
  WB2_TRY(pk.commit());

  DetParams p;
  p.f = f; p.t = t; p.c = c; p.g = g;
  p.off_f = pk.dev<int64_t>(o_f);
  p.off_t = pk.dev<int64_t>(o_t);
  p.off_c = off_c ? pk.dev<int64_t>(o_c) : nullptr;
  p.off_g = off_g ? pk.dev<int64_t>(o_g) : nullptr;
  wu.bind(p);
  p.partial = pk.dev<double>(o_part);
  p.rows_per_block = br.rows_per_block; p.nblk = br.nblk;

  const bool weighted = w->col_w != nullptr || w->cell_w != nullptr;

  // Fast path: TMA-staged persistent kernels (det_tma.cu) when every slab is
  // 16-byte aligned and the weights are separable: one column segment, or
  // several (lane-contiguous column spans, for many regions).
  // WB2_DET_PATH=ldg forces the LDG kernel (A/B measurements, tests).
  const char* force = getenv("WB2_DET_PATH");
  const bool want_tma = !(force && strcmp(force, "ldg") == 0);
  if (want_tma && dtype == WB2_F32 && vec_ok && !weighted && w->ncol % 4 == 0 &&
      mode != MODE_VECTOR) {
    const int trc =
        w->nseg == 1
            ? det_metrics_tma(ctx, mode == MODE_CLIM, f, t, c, nfield, p.off_f, p.off_t,
                              p.off_c, p.row_w, p.seg_w, w, skipna, out)
            : det_metrics_tma_seg(ctx, mode == MODE_CLIM, f, t, c, nfield, p.off_f, p.off_t,
                                  p.off_c, w, skipna, out);
    if (trc < 0) return trc;
    if (trc == 1) {
      WB2_TRY(pk.release());
      return WB2_OK;
    }
  }

  int rc = dtype == WB2_F32
               ? launch_dtype<float>(ctx, p, nfield, mode, skipna != 0, weighted, vec_ok)
               : launch_dtype<double>(ctx, p, nfield, mode, skipna != 0, weighted, vec_ok);
  if (rc != WB2_OK) return rc;
  WB2_TRY(launch_block_sum(ctx, p.partial, out, nfield, br.nblk, static_cast<int>(per_field)));
  ctx->launches += 2;
  WB2_TRY(pk.release());
  return WB2_OK;
}

}  // namespace wb2

using namespace wb2;

extern "C" {

int wb2_det_metrics(wb2_ctx* ctx, const void* f, const void* t, const void* c, int dtype,
                    int64_t nfield, const int64_t* off_f, const int64_t* off_t,
                    const int64_t* off_c, const wb2_weights* w, int skipna, double* out) {
  WB2_NVTX("wb2_det_metrics");
  return det_metrics_impl(ctx, c ? MODE_CLIM : MODE_PLAIN, f, t, c, nullptr, dtype, nfield,
                          off_f, off_t, c ? off_c : nullptr, nullptr, w, skipna, out);
}

int wb2_det_metrics_vector(wb2_ctx* ctx, const void* fu, const void* fv, const void* tu,
                           const void* tv, int dtype, int64_t nfield, const int64_t* off_fu,
                           const int64_t* off_fv, const int64_t* off_tu,
                           const int64_t* off_tv, const wb2_weights* w, int skipna,
                           double* out) {
  WB2_NVTX("wb2_det_metrics_vector");
  // operand order inside the kernel: f = fu, t = tu, c = fv, g = tv
  return det_metrics_impl(ctx, MODE_VECTOR, fu, tu, fv, tv, dtype, nfield, off_fu, off_tu,
                          off_fv, off_tv, w, skipna, out);
}

}  // extern "C"

// K9 -- SEEPS (Stable Equitable Error in Probability Space) maps (sm_90a).
//
// Replaces SpatialSEEPS.compute_chunk (weatherbench2/metrics.py:417-513): both
// forecast and truth precipitation are put into the categories dry / light /
// heavy with the reference's own comparisons (:449-454)
//     dry = x < dry_thr;  light = x > dry_thr and x < wet;  heavy = x >= wet
// (a value equal to dry_thr is in no category, and with wet < dry_thr a value
// can be in two: the score is the double sum  sum_fc sum_tc F[fc] T[tc] S[fc][tc]
// exactly like the reference's contingency-table dot product, :476-500), the
// 3 x 3 scoring matrix comes from the climatological dry fraction p1 of the
// cell (:482-492), and cells with p1 outside (min_p1, max_p1) are NaN
// (:503-504).  Like K6 the kernel can average `ngroup` time steps into one
// output map (Metric.compute, :117-138).  SEEPS itself (the spatial mean with
// skipna = True, :516-528) is K1 applied to these maps.
//
// Numerics follow NumPy's promotion, operand by operand, so that every map is
// float32(reference):
// - f, t, wet and p1 are read in their own dtypes (float32 or float64).  A
//   comparison runs in the promoted dtype of its two sides; widening to double
//   is exact, so all comparisons run in double.  The Python-float dry threshold
//   is a weak scalar: it is rounded to the precipitation operand's dtype, and
//   min_p1 / max_p1 to p1's.
// - The scoring matrix is formed in p1's dtype with the reference's operations
//   in its order, each rounded separately (explicit _rn intrinsics: nothing is
//   contracted), then widened.
// - The score is the reference's dot product in double: every entry of the
//   table times its matrix entry, so 0 * inf is NaN as in xr.dot.  The time
//   mean accumulates these double values and rounds once, to the float32 map.
//
// One thread per grid cell of an output map; 8 B (float32) or 16 B (float64)
// read (+ the wet-threshold slab, usually L2-resident) and 4 / ngroup bytes
// written per cell.
#include "common.cuh"

namespace wb2 {

constexpr int kSeepsThreads = 256;

struct SeepsParams {
  const void* f;
  const void* t;
  const void* wet;    // climatological wet threshold slabs
  const void* p1;     // [nrow][ncol] mean dry fraction
  float* out;         // [nout][nrow][ncol]
  const int64_t* off_f;   // [nout][ngroup]
  const int64_t* off_t;
  const int64_t* off_wf;  // wet threshold at the forecast's valid time
  const int64_t* off_wt;  // ... at the truth's valid time
  int64_t row_stride, wet_row_stride, cells_per_map;
  int32_t ngroup, nrow, ncol, bpm;
  int32_t f_f64, t_f64, wet_f64;
  double dry_f, dry_t;    // the dry threshold in the forecast's / truth's dtype
  double min_p1, max_p1;  // in p1's dtype
};

__device__ __forceinline__ double seeps_ld_stream(const void* p, int f64, int64_t i) {
  return f64 ? ldg_stream(static_cast<const double*>(p) + i)
             : double(ldg_stream(static_cast<const float*>(p) + i));
}

__device__ __forceinline__ double seeps_ld(const void* p, int f64, int64_t i) {
  return f64 ? __ldg(static_cast<const double*>(p) + i)
             : double(__ldg(static_cast<const float*>(p) + i));
}

// category membership flags (bit 0 dry, 1 light, 2 heavy); NaN -> -1
__device__ __forceinline__ int seeps_cat(double x, double dry, double wet) {
  if (!(x == x)) return -1;
  int c = 0;
  if (x < dry) c |= 1;
  if (x > dry && x < wet) c |= 2;
  if (x >= wet) c |= 4;
  return c;
}

// correctly rounded arithmetic in p1's dtype
__device__ __forceinline__ float s_add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float s_sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float s_mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float s_div(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double s_add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double s_sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double s_mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double s_div(double a, double b) { return __ddiv_rn(a, b); }

// 0.5 * scoring matrix, S[forecast_cat][truth_cat] (:487-499), in P
template <typename P>
__device__ __forceinline__ void seeps_matrix(P p1, double S[3][3]) {
  const P h = P(0.5), one = P(1), q1 = s_sub(one, p1), q2 = s_add(P(2), p1);
  const P inv_p1 = s_div(one, p1), c3 = s_div(P(3), q2);
  S[0][0] = 0.0;
  S[0][1] = double(s_mul(h, s_div(one, q1)));
  S[0][2] = double(s_mul(h, s_div(P(4), q1)));
  S[1][0] = double(s_mul(h, inv_p1));
  S[1][1] = 0.0;
  S[1][2] = double(s_mul(h, s_div(P(3), q1)));
  S[2][0] = double(s_mul(h, s_add(inv_p1, c3)));
  S[2][1] = double(s_mul(h, c3));
  S[2][2] = 0.0;
}

template <bool SKIPNA, typename P>
__global__ void __launch_bounds__(kSeepsThreads) seeps_maps_kernel(const SeepsParams p) {
  const int64_t j = blockIdx.x / p.bpm;
  const int64_t ci = int64_t(blockIdx.x % p.bpm) * kSeepsThreads + threadIdx.x;
  if (ci >= p.cells_per_map) return;
  const int row = static_cast<int>(ci / p.ncol);
  const int col = static_cast<int>(ci % p.ncol);
  const int64_t cell = int64_t(row) * p.row_stride + col;
  const int64_t wcell = int64_t(row) * p.wet_row_stride + col;
  const double nanv = __longlong_as_double(0x7ff8000000000000ll);
  const P p1 = __ldg(static_cast<const P*>(p.p1) + ci);
  // :506-507, compared in p1's dtype (the bounds are already rounded to it)
  const bool masked = !(double(p1) < p.max_p1) || !(double(p1) > p.min_p1);
  double S[3][3];
  seeps_matrix<P>(p1, S);
  double acc = 0.0, last = 0.0;
  int cnt = 0;
  for (int g = 0; g < p.ngroup; ++g) {
    const int64_t field = j * p.ngroup + g;
    const double f = seeps_ld_stream(p.f, p.f_f64, p.off_f[field] + cell);
    const double t = seeps_ld_stream(p.t, p.t_f64, p.off_t[field] + cell);
    const double wf = seeps_ld(p.wet, p.wet_f64, p.off_wf[field] + wcell);
    const double wt = seeps_ld(p.wet, p.wet_f64, p.off_wt[field] + wcell);
    const int cf = seeps_cat(f, p.dry_f, wf);
    const int ct = seeps_cat(t, p.dry_t, wt);
    double v;
    if (cf < 0 || ct < 0 || masked) {
      v = nanv;
    } else {
      // xr.dot over the whole table: an unselected entry contributes 0 * S
      v = 0.0;
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b)
          v = __dadd_rn(v, __dmul_rn(double((cf >> a & 1) & (ct >> b & 1)), S[a][b]));
    }
    last = v;
    if (SKIPNA) {
      if (v == v) { acc += v; ++cnt; }
    } else {
      acc += v;
    }
  }
  double r;
  if (p.ngroup == 1) r = last;
  else if (SKIPNA) r = cnt > 0 ? acc / double(cnt) : nanv;
  else r = acc / double(p.ngroup);
  p.out[j * p.cells_per_map + ci] = __double2float_rn(r);
}

template <bool SKIPNA>
void seeps_launch(const SeepsParams& p, int p1_f64, dim3 grid, cudaStream_t s) {
  if (p1_f64) seeps_maps_kernel<SKIPNA, double><<<grid, kSeepsThreads, 0, s>>>(p);
  else seeps_maps_kernel<SKIPNA, float><<<grid, kSeepsThreads, 0, s>>>(p);
}

// a Python float compared with a float32 array is rounded to float32 first
inline double seeps_weak(double x, int dtype) {
  return dtype == WB2_F64 ? x : double(static_cast<float>(x));
}

}  // namespace wb2

using namespace wb2;

extern "C" int wb2_seeps_maps(wb2_ctx* ctx, const void* f, int f_dtype, const void* t,
                              int t_dtype, const void* wet, int wet_dtype, const void* p1,
                              int p1_dtype, int64_t nout, int32_t ngroup,
                              const int64_t* off_f, const int64_t* off_t,
                              const int64_t* off_wet_f, const int64_t* off_wet_t, int32_t nrow,
                              int32_t ncol, int64_t row_stride, int64_t wet_row_stride,
                              double dry_threshold, double min_p1, double max_p1, int skipna,
                              float* out) {
  WB2_NVTX("wb2_seeps_maps");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_REQUIRE(nrow > 0 && ncol > 0 && row_stride >= ncol && wet_row_stride >= ncol,
              "bad grid: nrow=%d ncol=%d", nrow, ncol);
  WB2_REQUIRE(nout >= 0 && ngroup >= 1, "nout must be >= 0 and ngroup >= 1");
  for (const int dt : {f_dtype, t_dtype, wet_dtype, p1_dtype})
    WB2_REQUIRE(dt == WB2_F32 || dt == WB2_F64, "dtype must be WB2_F32 or WB2_F64, got %d", dt);
  if (nout == 0) return WB2_OK;
  WB2_REQUIRE(f && t && wet && p1 && out && off_f && off_t && off_wet_f && off_wet_t,
              "NULL argument");
  DeviceGuard guard(ctx->device);
  const int64_t nfield = nout * ngroup;
  Packer pk(ctx);
  const size_t o0 = pk.add(off_f, nfield * sizeof(int64_t));
  const size_t o1 = pk.add(off_t, nfield * sizeof(int64_t));
  const size_t o2 = pk.add(off_wet_f, nfield * sizeof(int64_t));
  const size_t o3 = pk.add(off_wet_t, nfield * sizeof(int64_t));
  WB2_TRY(pk.commit());
  SeepsParams p;
  p.f = f; p.t = t; p.wet = wet; p.p1 = p1; p.out = out;
  p.off_f = pk.dev<int64_t>(o0); p.off_t = pk.dev<int64_t>(o1);
  p.off_wf = pk.dev<int64_t>(o2); p.off_wt = pk.dev<int64_t>(o3);
  p.row_stride = row_stride; p.wet_row_stride = wet_row_stride;
  p.cells_per_map = int64_t(nrow) * ncol;
  p.ngroup = ngroup; p.nrow = nrow; p.ncol = ncol;
  p.bpm = static_cast<int32_t>((p.cells_per_map + kSeepsThreads - 1) / kSeepsThreads);
  p.f_f64 = f_dtype == WB2_F64; p.t_f64 = t_dtype == WB2_F64; p.wet_f64 = wet_dtype == WB2_F64;
  p.dry_f = seeps_weak(dry_threshold, f_dtype);
  p.dry_t = seeps_weak(dry_threshold, t_dtype);
  p.min_p1 = seeps_weak(min_p1, p1_dtype);
  p.max_p1 = seeps_weak(max_p1, p1_dtype);
  WB2_REQUIRE(nout * int64_t(p.bpm) < (int64_t(1) << 31), "launch too large");
  const dim3 grid(static_cast<unsigned>(nout * p.bpm));
  if (skipna) seeps_launch<true>(p, p1_dtype == WB2_F64, grid, ctx->stream);
  else seeps_launch<false>(p, p1_dtype == WB2_F64, grid, ctx->stream);
  WB2_CUDA_TRY(cudaGetLastError());
  ctx->launches += 1;
  WB2_TRY(pk.release());
  return WB2_OK;
}

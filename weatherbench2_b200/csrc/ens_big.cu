// K2b -- ensemble metrics for LARGE ensembles (64 < M <= 1551), sm_90a.
//
// Same outputs as ens_metrics.cu (K2).  The register sorting network stops at
// 64 members; the reference's own tests use 100 and 1000
// (weatherbench2/metrics_test.py:785-789, 857-861).  Here a CTA stages a tile
// of 32 consecutive grid points x M members in shared memory with coalesced
// loads (padded to 33 columns: conflict-free both ways), then each warp takes
// points of the tile: lanes hold members m = lane, lane + 32, ...; the ordinal
// rank of a member is obtained by COUNTING (values smaller, plus equal values
// with a smaller index -- exactly np.argsort's stable order used at
// metrics.py:836-846, NaN last), O(M^2 / 32) per lane.  Correctness first: this
// path is for small grids; K2 is the fast path.
#include "region_reduce.cuh"

namespace wb2 {

constexpr int kBigWarps = 8;
constexpr int kBigThreads = kBigWarps * 32;
constexpr int kBigCols = 32;
constexpr int kBigPitch = kBigCols + 1;
constexpr int kBigStats = 5;

struct BigParams {
  const float* x;
  const float* t;
  const int64_t* off_x;
  const int64_t* off_t;
  const double* row_w;
  const int32_t* seg_start;
  const double* seg_w;
  const float* col_w;
  const float* cell_w;
  double* partial;  // [nfield][nblk][R][WB2_ENS_NSTAT]
  int64_t member_stride, row_stride;
  int32_t nmember, nrow, ncol, nregion, nseg, zero_skip, nblk, tiles_per_row;
  int32_t skipna;
};

// floats of the [M][33] tile, rounded up so the float64 area behind it is aligned
__host__ __device__ inline size_t big_tile_floats(int nmember) {
  return (size_t(nmember) * kBigPitch + 3) & ~size_t(3);
}

__device__ __forceinline__ bool big_less(float a, int ia, float b, int ib) {
  // total order of np.argsort (stable; NaN sorts last)
  const bool an = a != a, bn = b != b;
  if (an || bn) return an == bn ? ia < ib : bn;
  return a < b || (a == b && ia < ib);
}

__global__ void __launch_bounds__(kBigThreads) ens_big_kernel(const BigParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* tile = reinterpret_cast<float*>(smem_raw);                 // [M][33]
  double* red = reinterpret_cast<double*>(tile + big_tile_floats(p.nmember));
  // red: [warps][32 regions][10]
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int64_t field = blockIdx.x / p.nblk;
  const int blk = blockIdx.x % p.nblk;  // one (row, column tile) per block
  const int row = blk / p.tiles_per_row;
  const int col0 = (blk % p.tiles_per_row) * kBigCols;
  const int ncols = min(kBigCols, p.ncol - col0);
  const int M = p.nmember, R = p.nregion;
  const bool skipna = p.skipna != 0;
  const float* __restrict__ px = p.x + p.off_x[field] + int64_t(row) * p.row_stride + col0;
  const float* __restrict__ pt = p.t + p.off_t[field] + int64_t(row) * p.row_stride + col0;

  for (int m = warp; m < M; m += kBigWarps)
    if (lane < ncols) tile[m * kBigPitch + lane] = px[int64_t(m) * p.member_stride + lane];
  __syncthreads();

  double accd[WB2_ENS_NSTAT];
#pragma unroll
  for (int i = 0; i < WB2_ENS_NSTAT; ++i) accd[i] = 0.0;
  const float nanv = __int_as_float(0x7fc00000);
  const float fm = float(M);

  for (int c = warp; c < ncols; c += kBigWarps) {
    const int col = col0 + c;
    const float t = pt[c];
    // ---- moments and skill over the lane's members --------------------------
    float sumx = 0.f, suma = 0.f, nval = 0.f, naval = 0.f;
    for (int m = lane; m < M; m += 32) {
      const float xm = tile[m * kBigPitch + c];
      const float a = fabsf(t - xm);
      if (skipna) {
        if (xm == xm) { sumx += xm; nval += 1.f; }
        if (a == a) { suma += a; naval += 1.f; }
      } else {
        sumx += xm;
        suma += a;
      }
    }
    sumx = warp_sum(sumx); suma = warp_sum(suma);
    nval = warp_sum(nval); naval = warp_sum(naval);
    const float mean = skipna ? sumx / nval : sumx / fm;
    // ranks come from the raw tile values; each term is formed on the member
    // relative to the mean, as in K2 (ens_point.cuh): a finite mean only
    const bool finite_mean = fabsf(mean) <= __int_as_float(0x7f7fffff);
    const float shift = finite_mean ? mean : 0.f;
    float ss = 0.f, s = 0.f;
    for (int m = lane; m < M; m += 32) {
      const float xm = tile[m * kBigPitch + c];
      const float dx = xm - shift;
      if (!skipna || dx == dx) ss += dx * dx;
      // ordinal rank by counting (metrics.py:836-846)
      int rank = 1;
      for (int j = 0; j < M; ++j) rank += big_less(tile[j * kBigPitch + c], j, xm, m) ? 1 : 0;
      const float term = (2.f * float(rank) - fm - 1.f) * dx;  // metrics.py:808
      if (!skipna || xm == xm) s += term;
    }
    ss = warp_sum(ss);
    s = warp_sum(s);
    // the n valid ranks' coefficients add up to n (n - M) (skipna, see ens_point)
    if (skipna) s += shift * (nval * (nval - fm));
    float val[kBigStats];
    const float var = !finite_mean ? nanv
                      : skipna ? (nval > 1.f ? ss / (nval - 1.f) : nanv) : ss / (fm - 1.f);
    const float dm = t - mean;
    val[0] = skipna ? suma / naval : suma / fm;
    val[1] = M < 2 ? 0.f : (skipna ? 2.f * (s / nval) / (fm - 1.f) : 2.f * (s / fm) / (fm - 1.f));
    val[2] = dm * dm;
    val[3] = var;
    val[4] = dm * dm - var / fm;
    // ---- lane r = region r applies its weight --------------------------------
    if (lane < R) {
      int k = 0;
      while (k + 1 < p.nseg && p.seg_start[k + 1] <= col) ++k;
      double w = p.row_w[int64_t(lane) * p.nrow + row] * p.seg_w[lane * p.nseg + k];
      if (p.col_w) w *= double(p.col_w[col]);
      if (p.cell_w) w *= double(p.cell_w[int64_t(row) * p.ncol + col]);
      if (!(p.zero_skip && w == 0.0)) {
#pragma unroll
        for (int i = 0; i < kBigStats; ++i) {
          if (skipna) {
            if (val[i] == val[i]) { accd[i] += w * double(val[i]); accd[kBigStats + i] += w; }
          } else {
            accd[i] += w * double(val[i]);
            accd[kBigStats + i] += w;
          }
        }
      }
    }
  }
#pragma unroll
  for (int i = 0; i < WB2_ENS_NSTAT; ++i) red[(warp * 32 + lane) * WB2_ENS_NSTAT + i] = accd[i];
  __syncthreads();
  double* out = p.partial + (field * p.nblk + blk) * int64_t(R) * WB2_ENS_NSTAT;
  for (int idx = threadIdx.x; idx < R * WB2_ENS_NSTAT; idx += kBigThreads) {
    const int r = idx / WB2_ENS_NSTAT, i = idx % WB2_ENS_NSTAT;
    double v = 0.0;
    for (int w = 0; w < kBigWarps; ++w) v += red[(w * 32 + r) * WB2_ENS_NSTAT + i];
    out[idx] = v;
  }
}

int ens_metrics_big(wb2_ctx* ctx, const float* x, const float* t, int32_t nmember,
                    int64_t member_stride, int64_t nfield, const int64_t* off_x,
                    const int64_t* off_t, const wb2_weights* w, int skipna, double* out) {
  const size_t smem = big_tile_floats(nmember) * sizeof(float) +
                      size_t(kBigWarps) * 32 * WB2_ENS_NSTAT * sizeof(double);
  if (smem > 220 * 1024) {
    set_error("wb2_ens_metrics: at most %d ensemble members are supported (got %d)",
              static_cast<int>((220 * 1024 - kBigWarps * 32 * WB2_ENS_NSTAT * 8) /
                               (kBigPitch * 4)),
              nmember);
    return WB2_EUNSUPPORTED;
  }
  const int R = w->nregion;
  const int tiles_per_row = (w->ncol + kBigCols - 1) / kBigCols;
  const int nblk = w->nrow * tiles_per_row;
  WB2_REQUIRE(nfield * int64_t(nblk) < (int64_t(1) << 31), "launch too large");
  const size_t per_field = size_t(R) * WB2_ENS_NSTAT;
  Packer pk(ctx);
  size_t o_x = pk.add(off_x, nfield * sizeof(int64_t));
  size_t o_t = pk.add(off_t, nfield * sizeof(int64_t));
  const WeightUpload wu(pk, w);
  size_t o_part = pk.reserve(size_t(nfield) * nblk * per_field * sizeof(double));
  WB2_TRY(pk.commit());
  BigParams p;
  p.x = x; p.t = t;
  p.off_x = pk.dev<int64_t>(o_x); p.off_t = pk.dev<int64_t>(o_t);
  wu.bind(p);
  p.partial = pk.dev<double>(o_part);
  p.member_stride = member_stride;
  p.nmember = nmember;
  p.nblk = nblk; p.tiles_per_row = tiles_per_row; p.skipna = skipna ? 1 : 0;
  WB2_TRY(launch_kernel(ctx, ens_big_kernel, dim3(static_cast<unsigned>(nfield * nblk)),
                        kBigThreads, smem, p));
  WB2_TRY(launch_block_sum(ctx, p.partial, out, nfield, nblk, static_cast<int>(per_field)));
  ctx->launches += 2;
  WB2_TRY(pk.release());
  return WB2_OK;
}

}  // namespace wb2

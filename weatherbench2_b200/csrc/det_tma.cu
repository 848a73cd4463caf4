// K1 fast path -- TMA-staged persistent kernel (sm_90a).
//
// Same arithmetic and outputs as det_metrics_kernel (det_metrics.cu), but the
// slabs are moved HBM -> shared memory by the TMA engine (1-D bulk copies,
// `cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes`, SASS
// UBLKCP) into a ring of stages guarded by full/empty mbarriers, so the number
// of bytes in flight per SM (~140 KB) no longer depends on registers or
// occupancy.  One persistent CTA per SM:
//   warp 8   : producer -- one elected lane walks the CTA's tile list (32-bit
//              incremental index math only) and issues 2 or 3 bulk copies per
//              tile (forecast, truth[, clim]);
//   warps 0-7: consumers -- warp pair q = w/2 owns tiles q, q+4, ...; each warp
//              of the pair reads one half of the tile with conflict-free
//              LDS.128, accumulates the unweighted f32 sums, releases the
//              stage, butterfly-reduces and lets lane r add region r's float64
//              weight * sums to its accumulators.
// A tile is one whole row (5760 B per operand at 1440 columns), so the producer
// issues one tile per ~750 cycles at full HBM rate.  Tiles are dealt to CTAs in
// contiguous ranges, so a CTA touches few fields; every (CTA, warp) writes
// float64 partials per touched field and a finalize kernel adds them in a
// fixed order (deterministic).
//
// Eligibility (checked by the caller): float32, every slab 16-byte aligned
// (offsets, row stride and ncol multiples of 4 elements), one column segment,
// no per-column / per-cell weight factor.  Everything else takes the LDG kernel.
// det_tma_seg_kernel (second half of this file) is the variant for many regions.
#include <algorithm>

#include "region_reduce.cuh"
#include "tma_utils.cuh"

namespace wb2 {

constexpr int kConsumerWarps = 8;
constexpr int kTmaThreads = (kConsumerWarps + 1) * 32;
constexpr int kTilesInFlight = kConsumerWarps / 2;  // tiles being consumed at once

struct TmaParams {
  const float* f;
  const float* t;
  const float* c;
  const int64_t* off_f;
  const int64_t* off_t;
  const int64_t* off_c;
  const double* row_w;  // [R][nrow]
  const double* seg_w;  // [R][1]
  double* partial;      // [ncta][kConsumerWarps][maxslots][R][WB2_DET_NSTAT]
  int64_t ntiles;       // nfield * tiles_per_field
  int32_t nrow, ncol;
  int64_t row_stride;
  int32_t nregion;
  int32_t zero_skip;
  int32_t tiles_per_field;  // = nrow (one tile per row)
  int32_t nstage;           // multiple of kTilesInFlight
  int32_t stage_op_bytes;   // bytes reserved per operand per stage (128-B mult.)
  int32_t maxslots;
};

template <bool CLIM, bool SKIPNA>
__device__ __forceinline__ void tma_cell(float f, float t, float c, float* acc) {
  constexpr int NSUM = CLIM ? 6 : 3;
  const float d = f - t;
  if (SKIPNA) {
    if (d == d) {
      acc[0] += d * d;
      acc[1] += fabsf(d);
      acc[2] += d;
      acc[NSUM] += 1.0f;
    }
  } else {
    acc[0] += d * d;
    acc[1] += fabsf(d);
    acc[2] += d;
  }
  if (CLIM) {
    const float fa = f - c, ta = t - c;  // weatherbench2/metrics.py:405-406
    const float v3 = fa * ta, v4 = fa * fa, v5 = ta * ta;
    if (SKIPNA) {
      if (v3 == v3) { acc[3] += v3; acc[NSUM + 1] += 1.0f; }
      if (fa == fa) { acc[4] += v4; acc[NSUM + 2] += 1.0f; }
      if (ta == ta) { acc[5] += v5; acc[NSUM + 3] += 1.0f; }
    } else {
      acc[3] += v3;
      acc[4] += v4;
      acc[5] += v5;
    }
  }
}

// Persistent grid of the TMA kernels: ncta CTAs, each dealt a contiguous,
// balanced range of the tiles and so touching at most `maxslots` fields (the
// field slots of its float64 partials).
struct TmaGrid {
  int ncta, maxslots;
};
static TmaGrid tma_grid(const wb2_ctx* ctx, int64_t ntiles, int tiles_per_field) {
  int ncta = ctx->num_sms;
  if (ntiles < ncta) ncta = static_cast<int>(ntiles);
  const int64_t per = (ntiles + ncta - 1) / ncta;
  return {ncta, static_cast<int>((per + tiles_per_field - 1) / tiles_per_field) + 1};
}

// full / empty mbarriers of the stage ring; both warps of the consuming pair
// release a stage
__device__ __forceinline__ void init_ring(uint64_t* full, uint64_t* empty, int nstage) {
  if (threadIdx.x == 0) {
    for (int s = 0; s < nstage; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 2);
    }
    mbar_fence_init();
  }
}

// The single-lane TMA producer: streams the CTA's `ntiles` tiles (one row of
// forecast, truth[, climatology] each), starting at `row` of `field`, through
// the ring of `nstage` stages.
template <bool CLIM, typename P>
__device__ __forceinline__ void produce_rows(const P& p, unsigned char* smem, size_t stage_bytes,
                                             int nstage, uint64_t* full, uint64_t* empty,
                                             int64_t field, int row, int64_t ntiles) {
  constexpr int NOPER = CLIM ? 3 : 2;
  const float* pf = p.f + p.off_f[field];
  const float* pt = p.t + p.off_t[field];
  const float* pc = CLIM ? p.c + p.off_c[field] : nullptr;
  const uint32_t bytes = static_cast<uint32_t>(p.ncol) * 4u;
  int s = 0;
  uint32_t use = 0;
  for (int64_t j = 0; j < ntiles; ++j) {
    if (use > 0) mbar_wait(&empty[s], (use - 1) & 1);
    const int64_t e = int64_t(row) * p.row_stride;
    unsigned char* dst = smem + stage_bytes * s;
    mbar_arrive_expect_tx(&full[s], bytes * NOPER);
    tma_load_1d(dst, pf + e, bytes, &full[s]);
    tma_load_1d(dst + p.stage_op_bytes, pt + e, bytes, &full[s]);
    if (CLIM) tma_load_1d(dst + 2 * p.stage_op_bytes, pc + e, bytes, &full[s]);
    if (++s == nstage) { s = 0; ++use; }
    if (++row == p.nrow) {
      row = 0;
      ++field;
      if (j + 1 < ntiles) {
        pf = p.f + p.off_f[field];
        pt = p.t + p.off_t[field];
        if (CLIM) pc = p.c + p.off_c[field];
      }
    }
  }
}

template <bool CLIM, bool SKIPNA>
__global__ void __launch_bounds__(kTmaThreads, 1) det_tma_kernel(const TmaParams p) {
  constexpr int NOPER = CLIM ? 3 : 2;
  constexpr int NSUM = CLIM ? 6 : 3;
  // without skipna the weight sum is the plain cell count of the tile
  constexpr int NCNT = SKIPNA ? (CLIM ? 4 : 1) : 0;
  constexpr int NS = NSUM + NCNT;

  extern __shared__ __align__(128) unsigned char smem[];
  const int nstage = p.nstage;
  const size_t stage_bytes = size_t(NOPER) * p.stage_op_bytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + stage_bytes * nstage);
  uint64_t* empty = full + nstage;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  init_ring(full, empty, nstage);
  __syncthreads();

  // contiguous, balanced tile range of this CTA
  const int64_t per = p.ntiles / gridDim.x, extra = p.ntiles % gridDim.x;
  const int64_t b = blockIdx.x;
  const int64_t t0 = b * per + (b < extra ? b : extra);
  const int64_t t1 = t0 + per + (b < extra ? 1 : 0);
  const int64_t ncta_tiles = t1 - t0;
  const int64_t first_field = t0 / p.tiles_per_field;

  if (warp == kConsumerWarps) {
    // ------------------------------ producer --------------------------------
    if (lane == 0)
      produce_rows<CLIM>(p, smem, stage_bytes, nstage, full, empty, first_field,
                         static_cast<int>(t0 - first_field * p.tiles_per_field), ncta_tiles);
    return;
  }

  // -------------------------------- consumers --------------------------------
  const int R = p.nregion;
  const bool zero_skip = p.zero_skip != 0;
  double accd[NS + 1];  // [NS] = weight sum when !SKIPNA
#pragma unroll
  for (int i = 0; i <= NS; ++i) accd[i] = 0.0;
  int64_t cur_field = -1;

  auto flush_field = [&](int64_t field) {
    // lane r holds region r's sums of `field`; write them in public layout
    if (field < 0) return;
    const int slot = static_cast<int>(field - first_field);
    if (lane < R) {
      double* out = p.partial +
                    (((int64_t(blockIdx.x) * kConsumerWarps + warp) * p.maxslots + slot) * R +
                     lane) * WB2_DET_NSTAT;
#pragma unroll
      for (int st = 0; st < WB2_DET_NSTAT; ++st) {
        const int slot = k1_slot(st, NSUM, CLIM, SKIPNA);
        out[st] = slot >= 0 ? accd[slot] : 0.0;
      }
    }
#pragma unroll
    for (int i = 0; i <= NS; ++i) accd[i] = 0.0;
  };

  const int pair = warp >> 1, half = warp & 1;
  const int n4 = p.ncol >> 2;
  const int n4a = (n4 + 1) >> 1;
  const int i0 = half ? n4a : 0, i1 = half ? n4 : n4a;
  int64_t field = first_field;
  int row = static_cast<int>(t0 - first_field * p.tiles_per_field) + pair;
  int s = pair;
  uint32_t use = 0;
  for (int64_t j = pair; j < ncta_tiles; j += kTilesInFlight) {
    while (row >= p.nrow) { row -= p.nrow; ++field; }
    if (field != cur_field) {
      flush_field(cur_field);
      cur_field = field;
    }
    // region weight of this row (issued early, consumed after the tile)
    double w = 0.0;
    if (lane < R) w = p.row_w[int64_t(lane) * p.nrow + row] * p.seg_w[lane];

    const unsigned char* src = smem + stage_bytes * s;
    const float4* sf = reinterpret_cast<const float4*>(src);
    const float4* st = reinterpret_cast<const float4*>(src + p.stage_op_bytes);
    const float4* sc = reinterpret_cast<const float4*>(src + 2 * p.stage_op_bytes);

    float acc[NS > 0 ? NS : 1];
#pragma unroll
    for (int i = 0; i < NS; ++i) acc[i] = 0.0f;

    mbar_wait(&full[s], use & 1);
#pragma unroll 2
    for (int i = i0 + lane; i < i1; i += 32) {
      const float4 a = sf[i];
      const float4 bq = st[i];
      float4 cq = make_float4(0.f, 0.f, 0.f, 0.f);
      if (CLIM) cq = sc[i];
      tma_cell<CLIM, SKIPNA>(a.x, bq.x, cq.x, acc);
      tma_cell<CLIM, SKIPNA>(a.y, bq.y, cq.y, acc);
      tma_cell<CLIM, SKIPNA>(a.z, bq.z, cq.z, acc);
      tma_cell<CLIM, SKIPNA>(a.w, bq.w, cq.w, acc);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);  // this warp is done with the stage

#pragma unroll
    for (int i = 0; i < NS; ++i) acc[i] = warp_sum(acc[i]);
    if (lane < R && !(zero_skip && w == 0.0)) {
#pragma unroll
      for (int i = 0; i < NS; ++i) accd[i] += w * double(acc[i]);
      if (!SKIPNA) accd[NS] += w * double((i1 - i0) * 4);
    }
    row += kTilesInFlight;
    s += kTilesInFlight;
    if (s >= nstage) { s -= nstage; ++use; }
  }
  flush_field(cur_field);
}

__global__ void det_tma_finalize_kernel(const double* __restrict__ partial,
                                        double* __restrict__ out, int64_t ntiles, int ncta,
                                        int tiles_per_field, int maxslots, int per_field,
                                        int nwarps) {
  const int64_t field = blockIdx.x;
  const int64_t tf0 = field * tiles_per_field, tf1 = tf0 + tiles_per_field;
  const int64_t per = ntiles / ncta, extra = ntiles % ncta;
  for (int i = threadIdx.x; i < per_field; i += blockDim.x) {
    double v = 0.0;
    for (int b = 0; b < ncta; ++b) {
      const int64_t t0 = int64_t(b) * per + (b < extra ? b : extra);
      const int64_t t1 = t0 + per + (b < extra ? 1 : 0);
      if (t1 <= tf0 || t0 >= tf1) continue;
      const int slot = static_cast<int>(field - t0 / tiles_per_field);
      for (int w = 0; w < nwarps; ++w)
        v += partial[((int64_t(b) * nwarps + w) * maxslots + slot) * per_field + i];
    }
    out[field * per_field + i] = v;
  }
}

// Returns 1 if the TMA path ran, 0 if the launch is not eligible, < 0 on error.
int det_metrics_tma(wb2_ctx* ctx, bool clim, const void* f, const void* t, const void* c,
                    int64_t nfield, const int64_t* d_off_f, const int64_t* d_off_t,
                    const int64_t* d_off_c, const double* d_row_w, const double* d_seg_w,
                    const wb2_weights* w, int skipna, double* out) {
  const int noper = clim ? 3 : 2;
  if (w->ncol * 4 < 512) return 0;
  const int stage_op_bytes = (w->ncol * 4 + 127) / 128 * 128;
  const size_t budget = 220 * 1024;  // of the 227 KB a CTA may use on sm_90
  int nstage = static_cast<int>(budget / (size_t(noper) * stage_op_bytes));
  nstage = nstage / kTilesInFlight * kTilesInFlight;
  if (nstage > 32) nstage = 32;
  if (nstage < 2 * kTilesInFlight) return 0;
  const size_t smem = size_t(nstage) * noper * stage_op_bytes + 2 * nstage * sizeof(uint64_t);

  TmaParams p;
  p.f = static_cast<const float*>(f);
  p.t = static_cast<const float*>(t);
  p.c = static_cast<const float*>(c);
  p.off_f = d_off_f; p.off_t = d_off_t; p.off_c = d_off_c;
  p.row_w = d_row_w; p.seg_w = d_seg_w;
  p.nrow = w->nrow; p.ncol = w->ncol; p.row_stride = w->row_stride;
  p.nregion = w->nregion; p.zero_skip = w->zero_skip;
  p.tiles_per_field = w->nrow;
  p.ntiles = nfield * p.tiles_per_field;
  p.nstage = nstage; p.stage_op_bytes = stage_op_bytes;
  const TmaGrid g = tma_grid(ctx, p.ntiles, p.tiles_per_field);
  const int ncta = g.ncta;
  p.maxslots = g.maxslots;
  const size_t per_field = size_t(w->nregion) * WB2_DET_NSTAT;
  const size_t part_bytes = size_t(ncta) * kConsumerWarps * p.maxslots * per_field * sizeof(double);
  WB2_TRY(grow_buffer(ctx, ctx->tma_partial, ctx->tma_partial_cap, part_bytes));
  p.partial = ctx->tma_partial;
  WB2_CUDA_TRY(cudaMemsetAsync(p.partial, 0, part_bytes, ctx->stream));

  auto go = [&](auto kernel) { return launch_kernel(ctx, kernel, ncta, kTmaThreads, smem, p); };
  int rc;
  if (clim) rc = skipna ? go(det_tma_kernel<true, true>) : go(det_tma_kernel<true, false>);
  else rc = skipna ? go(det_tma_kernel<false, true>) : go(det_tma_kernel<false, false>);
  if (rc != WB2_OK) return rc;
  det_tma_finalize_kernel<<<static_cast<unsigned>(nfield), 128, 0, ctx->stream>>>(
      p.partial, out, p.ntiles, ncta, p.tiles_per_field, p.maxslots,
      static_cast<int>(per_field), kConsumerWarps);
  WB2_CUDA_TRY(cudaGetLastError());
  ctx->launches += 2;
  return 1;
}

// ---------------------------------------------------------------------------
// K1 fast path for MANY REGIONS -- TMA-staged persistent kernel with
// lane-contiguous column spans (sm_90a).
//
// The official WB2 evaluation runs 13-16 regions (scripts/evaluate.py:345-395);
// their longitude boxes cut a row into ~15 column segments.  Reducing every
// (row, segment) across the warp (det_metrics.cu / det_tma.cu) then costs more
// than the arithmetic.  Here the tile already sits in shared memory (same TMA
// ring as det_tma.cu), so a lane can own a CONTIGUOUS span of columns -- the
// SAME span, hence the same column segment, in every row.  The weights
// factorise as  W_r(row, seg) = row_c[row] * pattern[band(row)][r] * seg_w[seg][r]
// where the region pattern is constant over a BAND of consecutive rows (the
// latitude boxes), so the per-row work is only  band_acc += row_c[row] * partial
// (7 FMAs per span); the regions are applied to the band accumulators when the
// band changes, every 16 tiles and at field changes, warp-reduced into
// float64 shared-memory accumulators.  (v2 applied all regions at every span
// end: 16 x 8 FMAs per 11 cells, as much work as the cells themselves, and 112
// accumulator registers: 0.53 of the HBM roofline.)  Fields are flushed to
// per-(CTA, warp, field) float64 partials which det_tma_finalize_kernel adds in
// a fixed order.  Span width is odd so the scalar LDS of a warp are
// conflict-free.
//
// Eligibility: float32, 16-byte aligned slabs, no per-column / per-cell weight
// factor, nregion <= RCH (16; 8 with skipna) -- the host splits longer region
// lists into several launches.

// Consumer warps per CTA (CW in the kernel): 2 warps share a tile (half a row
// each), so CW / 2 tiles are consumed at once.  The kernel is partly
// latency-bound (dependent LDS -> FMA chains): 16 warps measured 3-7 % faster
// than 8 in one run, but that shape has seen far less testing, so it stays 8.
constexpr int kSegWarps = 8;
// regions per launch (RCH in the kernel); longer region lists take several
constexpr int seg_regions(bool skipna) { return skipna ? 8 : 16; }
constexpr int kSegDump = 16;  // tiles between band accumulator -> float64 dumps
constexpr int kSegMaxBands = 128;  // row bands (runs of equal region patterns)
constexpr int kSegMaxSpans = 64;  // spans per half row (two rounds of 32 lanes)

struct TmaSegParams {
  const float* f;
  const float* t;
  const float* c;
  const int64_t* off_f;
  const int64_t* off_t;
  const int64_t* off_c;
  const float* row_c;        // [nrow] common row factor (max_r |row_w[r][row]|)
  const int32_t* row_band;   // [nrow] band of the row (runs of equal region patterns)
  const float* pat;          // [nband][RCH] row_w[r][row] / row_c[row], zero padded
  int32_t nband;
  const float* seg_wf;       // [nseg][RCH] float32, zero padded
  const int32_t* seg_start;  // [nseg + 1]
  const int4* spans;         // [2][kSegMaxSpans] (first col, end col, segment, -)
  int32_t nspan[2];          // spans of the left / right half row
  double* partial;           // [ncta][warps][maxslots][R][WB2_DET_NSTAT]
  int64_t ntiles;
  int32_t nrow, ncol;
  int64_t row_stride;
  int32_t nregion, nseg;
  int32_t zero_skip;
  int32_t nstage;
  int32_t stage_op_bytes;
  int32_t maxslots;
};

template <bool CLIM, bool SKIPNA>
__global__ void __launch_bounds__(((kSegWarps + 1) * 32), 1)
    det_tma_seg_kernel(const TmaSegParams p) {
  constexpr int CW = kSegWarps, RCH = seg_regions(SKIPNA);
  constexpr int NOPER = CLIM ? 3 : 2;
  constexpr int NSUM = CLIM ? 6 : 3;
  // per-piece values: sums, then counts (skipna) or one cell count (!skipna)
  constexpr int NCNT = SKIPNA ? (CLIM ? 4 : 1) : 1;
  constexpr int NS = NSUM + NCNT;

  extern __shared__ __align__(128) unsigned char smem[];
  const int nstage = p.nstage;
  const size_t stage_bytes = size_t(NOPER) * p.stage_op_bytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + stage_bytes * nstage);
  uint64_t* empty = full + nstage;
  double* dacc = reinterpret_cast<double*>(empty + nstage);  // [warps][RCH][NS]
  float* s_segw = reinterpret_cast<float*>(dacc + CW * RCH * NS);  // [nseg][RCH]
  int* s_segstart = reinterpret_cast<int*>(s_segw + size_t(p.nseg) * RCH);       // [nseg + 1]
  float* s_pat = reinterpret_cast<float*>(s_segstart + p.nseg + 1);               // [nband][RCH]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  init_ring(full, empty, nstage);
  for (int i = threadIdx.x; i < p.nseg * RCH; i += ((CW + 1) * 32)) s_segw[i] = p.seg_wf[i];
  for (int i = threadIdx.x; i <= p.nseg; i += ((CW + 1) * 32)) s_segstart[i] = p.seg_start[i];
  for (int i = threadIdx.x; i < p.nband * RCH; i += ((CW + 1) * 32)) s_pat[i] = p.pat[i];
  for (int i = threadIdx.x; i < CW * RCH * NS; i += ((CW + 1) * 32)) dacc[i] = 0.0;
  __syncthreads();

  const int64_t per = p.ntiles / gridDim.x, extra = p.ntiles % gridDim.x;
  const int64_t b = blockIdx.x;
  const int64_t t0 = b * per + (b < extra ? b : extra);
  const int64_t t1 = t0 + per + (b < extra ? 1 : 0);
  const int64_t ncta_tiles = t1 - t0;
  const int64_t first_field = t0 / p.nrow;

  if (warp == CW) {
    // ------------------------------ producer --------------------------------
    if (lane == 0)
      produce_rows<CLIM>(p, smem, stage_bytes, nstage, full, empty, first_field,
                         static_cast<int>(t0 - first_field * p.nrow), ncta_tiles);
    return;
  }

  // -------------------------------- consumers --------------------------------
  const int R = p.nregion;
  const bool zero_skip = p.zero_skip != 0;
  const int pair = warp >> 1, half = warp & 1;
  // Host-built spans of this half row: contiguous column ranges that never
  // cross a segment boundary, at most 32 per round (one per lane), so the
  // region update below is warp-uniform.
  const int nspan = p.nspan[half];
  const int4* spans = p.spans + half * kSegMaxSpans;

  // A lane owns the same (at most two) column spans in every row, i.e. fixed
  // segments.  W_r(row, seg) = row_c[row] * pattern[band(row)][r] * seg_w[seg][r]
  // with the region pattern constant over a BAND of consecutive rows (the
  // latitude boxes of the regions), so the per-row work is only
  // band_acc += row_c[row] * part; the regions are applied when the band
  // changes, every kSegDump tiles and at field changes.
  int4 my_span[2];
  my_span[0] = lane < nspan ? spans[lane] : make_int4(0, 0, 0, 0);
  my_span[1] = lane + 32 < nspan ? spans[lane + 32] : make_int4(0, 0, 0, 0);
  float band_acc[2][NS];
#pragma unroll
  for (int k = 0; k < 2; ++k)
#pragma unroll
    for (int i = 0; i < NS; ++i) band_acc[k][i] = 0.f;
  double* my_dacc = dacc + warp * RCH * NS;
  int since_dump = 0;
  int cur_band = -1;
  int64_t cur_field = -1;

  auto dump = [&]() {
    // band accumulators -> regions -> float64 shared accumulators of this warp
    if (cur_band >= 0 && since_dump > 0) {
      const float* pat = s_pat + cur_band * RCH;
      const float* wv0 = s_segw + my_span[0].z * RCH;
      const float* wv1 = s_segw + my_span[1].z * RCH;
      for (int r = 0; r < R; ++r) {
        // a region that does not contain this band gets nothing (warp-uniform
        // test: most bands touch only a few of the regions)
        if (zero_skip && pat[r] == 0.f) continue;
        const float w0 = pat[r] * wv0[r], w1 = pat[r] * wv1[r];
        const bool use0 = my_span[0].y > my_span[0].x && (w0 != 0.f || !zero_skip);
        const bool use1 = my_span[1].y > my_span[1].x && (w1 != 0.f || !zero_skip);
        float mine = 0.f;  // lane i ends up with the total of statistic i
#pragma unroll
        for (int i = 0; i < NS; ++i) {
          float v = use0 ? w0 * band_acc[0][i] : 0.f;
          if (use1) v = fmaf(w1, band_acc[1][i], v);
          v = warp_sum(v);
          if (lane == i) mine = v;
        }
        if (lane < NS) my_dacc[r * NS + lane] += double(mine);
      }
    }
#pragma unroll
    for (int k = 0; k < 2; ++k)
#pragma unroll
      for (int i = 0; i < NS; ++i) band_acc[k][i] = 0.f;
    since_dump = 0;
    __syncwarp();
  };
  auto flush_field = [&](int64_t field) {
    if (field < 0) return;
    dump();
    const int slot = static_cast<int>(field - first_field);
    double* out = p.partial +
                  ((int64_t(blockIdx.x) * CW + warp) * p.maxslots + slot) *
                      int64_t(R) * WB2_DET_NSTAT;
    for (int idx = lane; idx < R * WB2_DET_NSTAT; idx += 32) {
      const int r = idx / WB2_DET_NSTAT;
      const int st = idx - r * WB2_DET_NSTAT;
      const int slot_i = k1_slot(st, NSUM, CLIM, SKIPNA);
      out[idx] = slot_i >= 0 ? my_dacc[r * NS + slot_i] : 0.0;
    }
    __syncwarp();
    for (int i = lane; i < RCH * NS; i += 32) my_dacc[i] = 0.0;
    __syncwarp();
  };

  int64_t field = first_field;
  int row = static_cast<int>(t0 - first_field * p.nrow) + pair;
  int s = pair;
  uint32_t use = 0;
  for (int64_t j = pair; j < ncta_tiles; j += (CW / 2)) {
    while (row >= p.nrow) { row -= p.nrow; ++field; }
    if (field != cur_field) {
      flush_field(cur_field);
      cur_field = field;
    }
    // common row factor and band of this row (broadcast loads, issued before
    // the wait)
    const float crow = __ldg(p.row_c + row);
    const int band = __ldg(p.row_band + row);
    if (band != cur_band) {
      dump();
      cur_band = band;
    }

    const unsigned char* src = smem + stage_bytes * s;
    const float* sf = reinterpret_cast<const float*>(src);
    const float* st_ = reinterpret_cast<const float*>(src + p.stage_op_bytes);
    const float* sc = reinterpret_cast<const float*>(src + 2 * p.stage_op_bytes);

    mbar_wait(&full[s], use & 1);
    if (crow != 0.f || !zero_skip) {  // rows outside every region: metrics.py:160
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const int4 sp = my_span[k];  // x = first column, y = end, z = segment
        float part[NS];
#pragma unroll
        for (int i = 0; i < NS; ++i) part[i] = 0.f;
#pragma unroll 4
        for (int col = sp.x; col < sp.y; ++col)
          tma_cell<CLIM, SKIPNA>(sf[col], st_[col], CLIM ? sc[col] : 0.f, part);
        if (!SKIPNA) part[NSUM] = float(sp.y - sp.x);
#pragma unroll
        for (int i = 0; i < NS; ++i) band_acc[k][i] = fmaf(crow, part[i], band_acc[k][i]);
      }
      ++since_dump;
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);

    if (since_dump >= kSegDump) dump();
    row += (CW / 2);
    s += (CW / 2);
    if (s >= nstage) { s -= nstage; ++use; }
  }
  flush_field(cur_field);
}

// Returns 1 if the kernel ran, 0 if not eligible, < 0 on error.  Handles the
// regions [r0, r0 + nreg) of `w`; `out` is the full [nfield][w->nregion][10]
// array (this launch fills only its regions).
static int launch_seg(wb2_ctx* ctx, bool clim, bool skipna, const TmaSegParams& p, int ncta,
                      size_t smem) {
  auto go = [&](auto kernel) {
    return launch_kernel(ctx, kernel, ncta, (kSegWarps + 1) * 32, smem, p);
  };
  if (clim) return skipna ? go(det_tma_seg_kernel<true, true>)
                          : go(det_tma_seg_kernel<true, false>);
  return skipna ? go(det_tma_seg_kernel<false, true>) : go(det_tma_seg_kernel<false, false>);
}

__global__ void seg_scatter_kernel(const double* __restrict__ tmp, double* __restrict__ out,
                                   int nreg, int r0, int rtotal) {
  // tmp [nfield][nreg][10] -> out [nfield][rtotal][10] at region offset r0
  const int64_t field = blockIdx.x;
  for (int i = threadIdx.x; i < nreg * WB2_DET_NSTAT; i += blockDim.x)
    out[(field * rtotal + r0) * WB2_DET_NSTAT + i] = tmp[field * nreg * WB2_DET_NSTAT + i];
}

int det_metrics_tma_seg(wb2_ctx* ctx, bool clim, const void* f, const void* t, const void* c,
                        int64_t nfield, const int64_t* d_off_f, const int64_t* d_off_t,
                        const int64_t* d_off_c, const wb2_weights* w, int skipna, double* out) {
  const int noper = clim ? 3 : 2;
  if (w->ncol * 4 < 512 || w->ncol % 4 != 0) return 0;
  constexpr int CW = kSegWarps;
  const int rch = seg_regions(skipna);
  const int nsum = clim ? 6 : 3;
  const int ns = nsum + (skipna ? (clim ? 4 : 1) : 1);
  const int stage_op_bytes = (w->ncol * 4 + 127) / 128 * 128;
  // Row bands per region chunk: runs of consecutive rows whose normalised region
  // pattern row_w[r][row] / max_r |row_w[r][row]| is the same for all regions
  // of the chunk (the latitude boxes).  Arbitrary per-row patterns (more than
  // kSegMaxBands runs) take the LDG path.
  struct ChunkBands {
    std::vector<float> row_c, pat;
    std::vector<int32_t> row_band;
    int nband = 0;
  };
  std::vector<ChunkBands> chunks;
  for (int r0 = 0; r0 < w->nregion; r0 += rch) {
    const int nreg = std::min(rch, w->nregion - r0);
    ChunkBands cb;
    cb.row_c.resize(w->nrow);
    cb.row_band.resize(w->nrow);
    std::vector<float> cur(rch, 0.f), prev(rch, 0.f);
    for (int i = 0; i < w->nrow; ++i) {
      double cmax = 0.0;
      for (int r = 0; r < nreg; ++r)
        cmax = std::max(cmax, std::fabs(w->row_w[size_t(r0 + r) * w->nrow + i]));
      for (int r = 0; r < rch; ++r)
        cur[r] = (r < nreg && cmax > 0.0)
                     ? static_cast<float>(w->row_w[size_t(r0 + r) * w->nrow + i] / cmax)
                     : 0.f;
      if (cb.nband == 0 || cur != prev) {
        if (cb.nband == kSegMaxBands) return 0;
        cb.pat.insert(cb.pat.end(), cur.begin(), cur.end());
        ++cb.nband;
        prev = cur;
      }
      cb.row_c[i] = static_cast<float>(cmax);
      cb.row_band[i] = cb.nband - 1;
    }
    chunks.push_back(std::move(cb));
  }
  const size_t fixed = size_t(CW) * rch * ns * sizeof(double) +
                       size_t(w->nseg) * rch * sizeof(float) + size_t(w->nseg + 1) * sizeof(int) +
                       size_t(kSegMaxBands) * rch * sizeof(float) + 256;
  const size_t budget = 220 * 1024;
  if (fixed >= budget) return 0;
  int nstage = static_cast<int>((budget - fixed) / (size_t(noper) * stage_op_bytes + 16));
  if (nstage > 32) nstage = 32;
  // CW / 2 stages are being consumed at any time; the rest is what the TMA
  // producer keeps in flight (>= 3 rows ~ 52 KB, above the ~44 KB per SM that
  // saturate HBM)
  if (nstage < CW / 2 + 3) return 0;
  const size_t smem = size_t(nstage) * noper * stage_op_bytes + 2 * nstage * sizeof(uint64_t) + fixed;

  const int64_t ntiles = nfield * w->nrow;
  const TmaGrid g = tma_grid(ctx, ntiles, w->nrow);
  const int ncta = g.ncta, maxslots = g.maxslots;

  // Boundary-aligned spans: every segment piece inside a half row is cut into
  // equal parts no longer than S columns, S the smallest length that keeps the
  // half row within 32 spans (one per lane); rows with very many tiny segments
  // take a second round.
  std::vector<int4> h_spans(2 * kSegMaxSpans, make_int4(0, 0, 0, 0));
  int h_nspan[2] = {0, 0};
  const int half_cols = (w->ncol + 1) / 2;
  for (int half = 0; half < 2; ++half) {
    const int h0 = half ? half_cols : 0, h1 = half ? w->ncol : half_cols;
    std::vector<int4> best;
    for (int limit : {32, kSegMaxSpans}) {
      for (int S = std::max(1, (h1 - h0 + limit - 1) / limit); S <= h1 - h0; ++S) {
        std::vector<int4> cur;
        for (int k = 0; k < w->nseg; ++k) {
          const int a = std::max(h0, w->seg_start[k]), b = std::min(h1, w->seg_start[k + 1]);
          if (a >= b) continue;
          const int parts = (b - a + S - 1) / S;
          for (int q = 0; q < parts; ++q) {
            const int c0 = a + int64_t(b - a) * q / parts, c1 = a + int64_t(b - a) * (q + 1) / parts;
            cur.push_back(make_int4(c0, c1, k, 0));
          }
        }
        if (static_cast<int>(cur.size()) <= limit) { best = cur; break; }
      }
      if (!best.empty()) break;
    }
    if (best.empty() && h1 > h0) return 0;  // too many segments: LDG path
    h_nspan[half] = static_cast<int>(best.size());
    for (size_t i = 0; i < best.size(); ++i) h_spans[half * kSegMaxSpans + i] = best[i];
  }

  // The tables of every region chunk go up in ONE Packer: the caller holds a
  // Packer slot (offset tables, weights) until this returns, and a Packer per
  // chunk would wrap the ring of kNumSlots slots at four chunks and overwrite
  // it while the kernels still read it.
  const int nchunk = static_cast<int>(chunks.size());
  std::vector<std::vector<float>> seg_wf(nchunk);
  std::vector<size_t> o_rc(nchunk), o_rb(nchunk), o_pat(nchunk), o_sw(nchunk);
  Packer pk(ctx);
  for (int ci = 0; ci < nchunk; ++ci) {
    const int r0 = ci * rch, nreg = std::min(rch, w->nregion - r0);
    // float32 weights of this region chunk
    seg_wf[ci].assign(size_t(w->nseg) * rch, 0.f);
    for (int r = 0; r < nreg; ++r)
      for (int k = 0; k < w->nseg; ++k)
        seg_wf[ci][size_t(k) * rch + r] =
            static_cast<float>(w->seg_w[size_t(r0 + r) * w->nseg + k]);
    const ChunkBands& cb = chunks[ci];
    o_rc[ci] = pk.add(cb.row_c.data(), cb.row_c.size() * sizeof(float));
    o_rb[ci] = pk.add(cb.row_band.data(), cb.row_band.size() * sizeof(int32_t));
    o_pat[ci] = pk.add(cb.pat.data(), cb.pat.size() * sizeof(float));
    o_sw[ci] = pk.add(seg_wf[ci].data(), seg_wf[ci].size() * sizeof(float));
  }
  const size_t o3 = pk.add(w->seg_start, size_t(w->nseg + 1) * sizeof(int32_t));
  const size_t o4 = pk.add(h_spans.data(), h_spans.size() * sizeof(int4));
  {
    // the first chunk has the most regions
    const size_t per_field = size_t(std::min(rch, w->nregion)) * WB2_DET_NSTAT;
    const size_t need = size_t(ncta) * CW * maxslots * per_field * sizeof(double) +
                        size_t(nfield) * per_field * sizeof(double);
    WB2_TRY(grow_buffer(ctx, ctx->tma_partial, ctx->tma_partial_cap, need));
  }
  WB2_TRY(pk.commit());

  for (int r0 = 0; r0 < w->nregion; r0 += rch) {
    const int ci = r0 / rch;
    const int nreg = std::min(rch, w->nregion - r0);
    const ChunkBands& cb = chunks[ci];
    const size_t per_field = size_t(nreg) * WB2_DET_NSTAT;
    const size_t part_bytes =
        size_t(ncta) * CW * maxslots * per_field * sizeof(double);

    TmaSegParams p;
    p.f = static_cast<const float*>(f);
    p.t = static_cast<const float*>(t);
    p.c = static_cast<const float*>(c);
    p.off_f = d_off_f; p.off_t = d_off_t; p.off_c = d_off_c;
    p.row_c = pk.dev<float>(o_rc[ci]); p.seg_wf = pk.dev<float>(o_sw[ci]);
    p.row_band = pk.dev<int32_t>(o_rb[ci]); p.pat = pk.dev<float>(o_pat[ci]);
    p.nband = cb.nband;
    p.seg_start = pk.dev<int32_t>(o3);
    p.spans = pk.dev<int4>(o4);
    p.nspan[0] = h_nspan[0]; p.nspan[1] = h_nspan[1];
    p.partial = ctx->tma_partial;
    p.ntiles = ntiles;
    p.nrow = w->nrow; p.ncol = w->ncol; p.row_stride = w->row_stride;
    p.nregion = nreg; p.nseg = w->nseg; p.zero_skip = w->zero_skip;
    p.nstage = nstage; p.stage_op_bytes = stage_op_bytes; p.maxslots = maxslots;
    WB2_CUDA_TRY(cudaMemsetAsync(p.partial, 0, part_bytes, ctx->stream));
    const int rc = launch_seg(ctx, clim, skipna, p, ncta, smem);
    if (rc != WB2_OK) return rc;
    double* tmp = reinterpret_cast<double*>(reinterpret_cast<char*>(ctx->tma_partial) + part_bytes);
    const bool direct = (nreg == w->nregion);
    det_tma_finalize_kernel<<<static_cast<unsigned>(nfield), 128, 0, ctx->stream>>>(
        p.partial, direct ? out : tmp, ntiles, ncta, w->nrow, maxslots,
        static_cast<int>(per_field), CW);
    WB2_CUDA_TRY(cudaGetLastError());
    ctx->launches += 2;
    if (!direct) {
      seg_scatter_kernel<<<static_cast<unsigned>(nfield), 128, 0, ctx->stream>>>(
          tmp, out, nreg, r0, w->nregion);
      WB2_CUDA_TRY(cudaGetLastError());
      ctx->launches += 1;
    }
  }
  WB2_TRY(pk.release());
  return 1;
}

}  // namespace wb2

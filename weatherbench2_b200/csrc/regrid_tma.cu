// K5 fast path -- conservative regridding with the source rows of a target
// group staged by TMA (sm_90a).
//
// Same arithmetic, tap order and outputs as regrid_kernel (regrid.cu), which
// replaces ConservativeRegridder.regrid_array (weatherbench2/regridding.py:
// 502-536).  Round-1 K5 ran at 0.61 of the HBM roofline: 25 thread
// instructions per source cell (issue 73 % busy) and 4.8 warps per issue stalled
// on the long scoreboard of its LDGs.  Two changes:
//   * the source rows a group of G target longitudes needs are CONTIGUOUS in
//     the (lon, lat) slab (one run, two at the periodic seam), so one elected
//     thread fetches the whole run with cp.async.bulk (SASS UBLKCP) into shared
//     memory, completion on an mbarrier; the 16-byte-aligned interior goes
//     through TMA, the <= 3 floats before / after it through plain loads.  Two
//     persistent CTAs per SM alternate between waiting for their run and
//     computing, so the copy of one overlaps the arithmetic of the other and no
//     warp ever waits on a global load;
//   * the contraction over source longitude walks each target's OWN taps (7 at
//     0.25 -> 1.5 degrees) instead of multiplying every staged row by a dense
//     G-wide weight vector (72 % of those FMAs had a zero weight): 5 thread
//     instructions per tap value, accumulators 3 instead of 12 registers.
// Stage 2 (contraction over source latitude + the NaN-aware division) is the
// same as in regrid_kernel, with the latitude CSR held in shared memory.
//
// Eligibility: source base 16-byte aligned, field stride a multiple of 4
// floats, every group's rows form at most two contiguous runs that fit the
// staging buffer, <= 1024 source latitudes.  Everything else takes regrid.cu.
#include <algorithm>

#include "common.cuh"
#include "tma_utils.cuh"

namespace wb2 {
namespace rgt {

constexpr int kThreads = 256;
constexpr int kMaxGroup = 4;  // target longitudes per work item (template G <= this)
constexpr int kMaxDpt = 4;   // source latitudes per thread
constexpr int kMaxSpans = 2;

struct GroupDesc {
  int32_t nspan;
  int32_t span_first[kMaxSpans];  // first element (row * nlat_s) of the run
  int32_t span_end[kMaxSpans];    // one past its last element
  int32_t span_base[kMaxSpans];   // shared-memory element where the ALIGNED run starts
  int32_t ntap[kMaxGroup];        // taps of target a: slots [a * maxtap, a * maxtap + ntap[a])
  float wsum[kMaxGroup];          // sum of target a's weights, added in tap order
  int32_t na;                     // targets in this group (<= G)
};

struct Tap {
  int32_t off;  // shared-memory element of the tap's source row
  float w;
};

struct Params {
  const float* src;
  float* dst;
  int64_t src_field_stride, dst_field_stride;
  const GroupDesc* groups;   // [ngroups]
  const Tap* taps;           // [ngroups][G * maxtap]
  const uint8_t* lon_nan;    // [nlon_t]
  const int32_t* lat_ptr;    // [nlat_t + 1]
  const int32_t* lat_idx;
  const float* lat_val;
  const uint8_t* lat_nan;    // [nlat_t]
  int32_t nlat_s, nlon_t, nlat_t;
  int32_t ngroups, maxtap, lat_nnz;
  int32_t stage_elems;       // floats reserved for the staged runs
  int64_t nitem;             // nfield * ngroups
};

// NTAP > 0: every target has exactly NTAP longitude taps (the regular grids:
// 7 at 0.25 -> 1.5 degrees) and the loops unroll completely; NTAP == 0: run-time
// tap counts.  LTAP likewise for the latitude taps of stage 2.
template <int DPT, int G, int NTAP>
__global__ void __launch_bounds__(kThreads, G <= 2 ? 4 : 2) regrid_tma_kernel(const Params p) {
  extern __shared__ __align__(128) unsigned char smem[];
  float* stg = reinterpret_cast<float*>(smem);
  float* ybuf = stg + p.stage_elems;                         // [G][2][nlat_s]
  // per-item descriptors, double buffered (the next item's are written while
  // the current item's are in use)
  GroupDesc* s_gd = reinterpret_cast<GroupDesc*>(ybuf + size_t(G) * 2 * p.nlat_s);
  Tap* s_tap = reinterpret_cast<Tap*>(s_gd + 2);             // [2][G * maxtap]
  uint64_t* full = reinterpret_cast<uint64_t*>(
      (reinterpret_cast<uintptr_t>(s_tap + 2 * G * p.maxtap) + 15) & ~uintptr_t(15));
  const int tid = threadIdx.x;
  const float nanv = __int_as_float(0x7fc00000);
  const int ntap_max = G * p.maxtap;

  if (tid == 0) {
    mbar_init(full, 1);
    mbar_fence_init();
  }
  __syncthreads();

  // Fetches the runs of `item` into the staging buffer -- TMA for the aligned
  // interior (thread 0), plain loads for the <= 3 + 3 floats around it -- and
  // its descriptors into slot `slot`.
  auto fetch = [&](int64_t item, int slot) {
    const int64_t field = item / p.ngroups;
    const int g = static_cast<int>(item - field * p.ngroups);
    const GroupDesc& gd = p.groups[g];
    const float* base = p.src + field * p.src_field_stride;  // 16-byte aligned
    if (tid == 0) {
      uint32_t bytes = 0;
      for (int k = 0; k < gd.nspan; ++k) {
        const int lo = (gd.span_first[k] + 3) & ~3, hi = gd.span_end[k] & ~3;
        if (hi > lo) bytes += uint32_t(hi - lo) * 4u;
      }
      mbar_arrive_expect_tx(full, bytes);
      for (int k = 0; k < gd.nspan; ++k) {
        const int lo = (gd.span_first[k] + 3) & ~3, hi = gd.span_end[k] & ~3;
        const int a0 = gd.span_first[k] & ~3;
        if (hi > lo)
          tma_load_1d(stg + gd.span_base[k] + (lo - a0), base + lo, uint32_t(hi - lo) * 4u, full);
      }
    } else if (tid >= 32 && tid < 32 + 8 * kMaxSpans) {
      const int k = (tid - 32) >> 3, j = (tid - 32) & 7;  // 4 head + 4 tail slots per run
      if (k < gd.nspan) {
        const int first = gd.span_first[k], end = gd.span_end[k];
        const int a0 = first & ~3;
        const int lo = min((first + 3) & ~3, end), hi = max(end & ~3, lo);
        const int e = j < 4 ? first + j : hi + (j - 4);
        const bool in = j < 4 ? e < lo : e < end;
        if (in) stg[gd.span_base[k] + (e - a0)] = __ldg(base + e);
      }
    } else if (tid >= 64 && tid < 64 + ntap_max) {
      s_tap[slot * ntap_max + (tid - 64)] = p.taps[size_t(g) * ntap_max + (tid - 64)];
    } else if (tid == 255) {
      s_gd[slot] = gd;
    }
  };

  int64_t item = blockIdx.x;
  if (item < p.nitem) fetch(item, 0);
  __syncthreads();
  uint32_t parity = 0;
  for (; item < p.nitem; item += gridDim.x) {
    const int64_t field = item / p.ngroups;
    const int g = static_cast<int>(item - field * p.ngroups);
    const int slot = static_cast<int>(parity);
    const GroupDesc& gd = s_gd[slot];
    const Tap* taps = s_tap + slot * ntap_max;
    const int na = gd.na;
    mbar_wait(full, parity);
    parity ^= 1u;

    // ---- stage 1: contract over source longitude, target by target ----------
    // y = sum_b W[a,b] x[b,d] WITHOUT looking at NaNs: a NaN anywhere in the
    // column poisons y, which is how the (rare) columns that need the NaN-aware
    // sums are found afterwards -- two instructions per tap value.
    for (int a = 0; a < na; ++a) {
      const int t0 = NTAP > 0 ? a * NTAP : a * p.maxtap;
      const int nt = NTAP > 0 ? NTAP : gd.ntap[a];
      float y[DPT];
#pragma unroll
      for (int i = 0; i < DPT; ++i) y[i] = 0.f;
      if (NTAP > 0) {
        Tap tp[NTAP > 0 ? NTAP : 1];
#pragma unroll
        for (int j = 0; j < NTAP; ++j) tp[j] = taps[t0 + j];
        float xv[NTAP > 0 ? NTAP : 1][DPT];
#pragma unroll
        for (int j = 0; j < NTAP; ++j)
#pragma unroll
          for (int i = 0; i < DPT; ++i) {
            const int d = tid + i * kThreads;
            xv[j][i] = (i + 1 < DPT || d < p.nlat_s) ? stg[tp[j].off + d] : 0.f;
          }
#pragma unroll
        for (int j = 0; j < NTAP; ++j)
#pragma unroll
          for (int i = 0; i < DPT; ++i) y[i] = fmaf(tp[j].w, xv[j][i], y[i]);
      } else {
        for (int j = 0; j < nt; ++j) {
          const Tap tp = taps[t0 + j];
#pragma unroll
          for (int i = 0; i < DPT; ++i) {
            const int d = tid + i * kThreads;
            const float xv = (i + 1 < DPT || d < p.nlat_s) ? stg[tp.off + d] : 0.f;
            y[i] = fmaf(tp.w, xv, y[i]);
          }
        }
      }
      const float ws = gd.wsum[a];
#pragma unroll
      for (int i = 0; i < DPT; ++i) {
        const int d = tid + i * kThreads;
        if (i + 1 < DPT || d < p.nlat_s) {
          float yy = y[i], v = ws;
          if (yy != yy) {  // a NaN (or Inf - Inf) in the column: the NaN-aware sums
            yy = 0.f;
            v = 0.f;
            for (int j = 0; j < nt; ++j) {
              const Tap tp = taps[t0 + j];
              const float xq = stg[tp.off + d];
              const bool ok = xq == xq;
              yy = fmaf(tp.w, ok ? xq : 0.f, yy);
              v = fmaf(tp.w, ok ? 1.f : 0.f, v);
            }
          }
          ybuf[(a * 2 + 0) * p.nlat_s + d] = yy;
          ybuf[(a * 2 + 1) * p.nlat_s + d] = v;
        }
      }
    }
    __syncthreads();  // staging consumed, ybuf complete
    if (item + gridDim.x < p.nitem) fetch(item + gridDim.x, slot ^ 1);

    // ---- stage 2: contract over source latitude, divide, store ---------------
    float* out = p.dst + field * p.dst_field_stride;
    const int a0 = g * G;
    const int nout = na * p.nlat_t;
    for (int o = tid; o < nout; o += kThreads) {
      const int al = o / p.nlat_t;
      const int c = o - al * p.nlat_t;
      float r;
      if (p.lon_nan[a0 + al] || p.lat_nan[c]) {
        r = nanv;
      } else {
        const float* yy = ybuf + size_t(al) * 2 * p.nlat_s;
        const float* vv = yy + p.nlat_s;
        float tot = 0.f, cnt = 0.f;
        const int l0 = __ldg(p.lat_ptr + c), l1 = __ldg(p.lat_ptr + c + 1);
#pragma unroll 8
        for (int tp = l0; tp < l1; ++tp) {
          const float w = __ldg(p.lat_val + tp);
          const int d = __ldg(p.lat_idx + tp);
          tot = fmaf(w, yy[d], tot);
          cnt = fmaf(w, vv[d], cnt);
        }
        r = tot / cnt;  // 0 / 0 -> NaN on purpose (regridding.py:534)
      }
      out[int64_t(a0 + al) * p.nlat_t + c] = r;
    }
    __syncthreads();  // ybuf (and the slots written by the next fetch) settle
  }
}

}  // namespace rgt

// 1 = handled, 0 = not eligible (the caller launches regrid_kernel), < 0 = error
template <int G>
static int regrid_tma_launch(wb2_ctx* ctx, const float* src, float* dst, int64_t nfield,
                             int64_t src_field_stride, int64_t dst_field_stride,
                             const wb2_csr* lon_w, const wb2_csr* lat_w) {
  using namespace rgt;
  if ((reinterpret_cast<uintptr_t>(src) & 15) != 0 || src_field_stride % 4 != 0) return 0;
  const int nlat_s = lat_w->n_src, nlon_t = lon_w->n_tgt, nlat_t = lat_w->n_tgt;
  if (nlat_s > kThreads * kMaxDpt) return 0;
  if (int64_t(lon_w->n_src) * nlat_s >= (int64_t(1) << 31)) return 0;
  const int ngroups = (nlon_t + G - 1) / G;
  std::vector<GroupDesc> groups(ngroups);
  int maxtap = 1, mintap = 1 << 30;
  for (int a = 0; a < nlon_t; ++a) {
    const int n = lon_w->row_ptr[a + 1] - lon_w->row_ptr[a];
    maxtap = std::max(maxtap, n);
    mintap = std::min(mintap, n);
  }
  if (G * maxtap > 128) return 0;  // descriptor copy uses threads 64 .. 191
  std::vector<Tap> taps(size_t(ngroups) * G * maxtap, Tap{0, 0.f});
  int stage_elems = 4;
  for (int g = 0; g < ngroups; ++g) {
    GroupDesc& gd = groups[g];
    const int a0 = g * G, a1 = std::min(nlon_t, a0 + G);
    gd.na = a1 - a0;
    std::vector<int> rows;
    for (int a = a0; a < a1; ++a)
      for (int tp = lon_w->row_ptr[a]; tp < lon_w->row_ptr[a + 1]; ++tp)
        rows.push_back(lon_w->col_idx[tp]);
    std::sort(rows.begin(), rows.end());
    rows.erase(std::unique(rows.begin(), rows.end()), rows.end());
    // contiguous runs of source rows
    int used = 0;
    std::vector<std::pair<int, int>> runs;  // [first row, last row]
    for (size_t i = 0; i < rows.size(); ++i) {
      if (!runs.empty() && rows[i] == runs.back().second + 1) runs.back().second = rows[i];
      else runs.push_back({rows[i], rows[i]});
    }
    if (runs.size() > size_t(kMaxSpans)) return 0;
    for (int k = 0; k < kMaxSpans; ++k) gd.span_first[k] = gd.span_end[k] = gd.span_base[k] = 0;
    for (size_t k = 0; k < runs.size(); ++k) {
      gd.span_first[k] = runs[k].first * nlat_s;
      gd.span_end[k] = (runs[k].second + 1) * nlat_s;
      gd.span_base[k] = used;
      const int a_lo = gd.span_first[k] & ~3;
      used += ((gd.span_end[k] - a_lo) + 3) & ~3;
    }
    gd.nspan = static_cast<int>(runs.size());
    stage_elems = std::max(stage_elems, used);
    // taps of target a at a * maxtap (uniform stride: the unrolled kernel
    // addresses them as a * NTAP with NTAP == maxtap)
    for (int a = a0; a < a1; ++a) {
      const int al = a - a0;
      float ws = 0.f;
      int nt = 0;
      for (int tp = lon_w->row_ptr[a]; tp < lon_w->row_ptr[a + 1]; ++tp, ++nt) {
        const int row = lon_w->col_idx[tp];
        int off = 0;
        for (size_t k = 0; k < runs.size(); ++k)
          if (row >= runs[k].first && row <= runs[k].second)
            off = gd.span_base[k] + (row * nlat_s - (gd.span_first[k] & ~3));
        taps[(size_t(g) * G + al) * maxtap + nt] = Tap{off, lon_w->val[tp]};
        ws = fmaf(lon_w->val[tp], 1.f, ws);
      }
      gd.wsum[al] = ws;
      gd.ntap[al] = nt;
    }
    for (int al = a1 - a0; al < kMaxGroup; ++al) {
      gd.wsum[al] = 0.f;
      gd.ntap[al] = 0;
    }
  }
  const size_t smem = size_t(stage_elems) * 4 + size_t(G) * 2 * nlat_s * 4 +
                      2 * sizeof(GroupDesc) + size_t(2) * G * maxtap * sizeof(Tap) + 32;
  // resident CTAs per SM the launch bounds promise: 4 (G <= 2) or 2
  if (smem > (G <= 2 ? 55 : 110) * 1024) return 0;

  const int lat_nnz = std::max(1, lat_w->row_ptr[nlat_t]);
  Packer pk(ctx);
  const size_t o0 = pk.add(groups.data(), groups.size() * sizeof(GroupDesc));
  const size_t o1 = pk.add(taps.data(), taps.size() * sizeof(Tap));
  const size_t o4 = pk.add(lon_w->nan_row, size_t(nlon_t));
  const size_t o5 = pk.add(lat_w->row_ptr, size_t(nlat_t + 1) * 4);
  const size_t o6 = pk.add(lat_w->col_idx, size_t(lat_nnz) * 4);
  const size_t o7 = pk.add(lat_w->val, size_t(lat_nnz) * 4);
  const size_t o8 = pk.add(lat_w->nan_row, size_t(nlat_t));
  WB2_TRY(pk.commit());
  Params p;
  p.src = src; p.dst = dst;
  p.src_field_stride = src_field_stride; p.dst_field_stride = dst_field_stride;
  p.groups = pk.dev<GroupDesc>(o0);
  p.taps = pk.dev<Tap>(o1);
  p.lon_nan = pk.dev<uint8_t>(o4);
  p.lat_ptr = pk.dev<int32_t>(o5); p.lat_idx = pk.dev<int32_t>(o6);
  p.lat_val = pk.dev<float>(o7); p.lat_nan = pk.dev<uint8_t>(o8);
  p.nlat_s = nlat_s; p.nlon_t = nlon_t; p.nlat_t = nlat_t;
  p.ngroups = ngroups; p.maxtap = maxtap; p.lat_nnz = lat_nnz;
  p.stage_elems = stage_elems;
  p.nitem = nfield * ngroups;
  const int64_t max_cta = int64_t(ctx->num_sms) * (G <= 2 ? 4 : 2);
  const unsigned grid = static_cast<unsigned>(std::min<int64_t>(p.nitem, max_cta));
  const int dpt = (nlat_s + kThreads - 1) / kThreads;
  const bool seven = mintap == 7 && maxtap == 7;  // the regular 6 : 1 coarsening
  auto go = [&](auto kernel) -> int {
    WB2_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      static_cast<int>(smem)));
    kernel<<<grid, kThreads, smem, ctx->stream>>>(p);
    WB2_CUDA_TRY(cudaGetLastError());
    return WB2_OK;
  };
  int rc;
  switch (dpt) {
    case 1: rc = go(regrid_tma_kernel<1, G, 0>); break;
    case 2: rc = go(regrid_tma_kernel<2, G, 0>); break;
    case 3: rc = seven ? go(regrid_tma_kernel<3, G, 7>) : go(regrid_tma_kernel<3, G, 0>); break;
    default: rc = go(regrid_tma_kernel<4, G, 0>); break;
  }
  if (rc != WB2_OK) return rc;
  ctx->launches += 1;
  WB2_TRY(pk.release());
  return 1;
}

int regrid_tma_try(wb2_ctx* ctx, const float* src, float* dst, int64_t nfield,
                   int64_t src_field_stride, int64_t dst_field_stride, const wb2_csr* lon_w,
                   const wb2_csr* lat_w) {
  const char* force = getenv("WB2_REGRID_PATH");
  if (force && strcmp(force, "ldg") == 0) return 0;
  // two targets per item; four when the two-target layout does not fit its shared memory
  int rc = regrid_tma_launch<2>(ctx, src, dst, nfield, src_field_stride, dst_field_stride, lon_w,
                                lat_w);
  if (rc == 0)
    rc = regrid_tma_launch<4>(ctx, src, dst, nfield, src_field_stride, dst_field_stride, lon_w,
                              lat_w);
  return rc;
}

}  // namespace wb2

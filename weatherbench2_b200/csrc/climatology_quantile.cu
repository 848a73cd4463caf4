// Day-of-year quantile and SEEPS climatologies: wb2_climatology_quantile (device
// series) and wb2_climatology_quantile_host (NumPy / memmap series, streamed in
// bands of cells through clim_stream_host).
//
// Replaces Quantile.compute and SEEPSThreshold.compute of
// scripts/compute_climatology.py:130-177 called from compute_rolling_stat
// (weatherbench2/utils.py:88-124), the `explicit` method: xarray's weighted
// type-7 quantile over (window, year) with the triangular window weights.  Per
// output value, after dropping NaN and zero-weight samples:
//   nw = (sum w)^2 / sum w^2,  c = [0, cumsum(w / sum w)] over the sorted values,
//   h = clip((nw - 1) q + 1, 1, nw),  v(c) = max((h-1)/nw, min(h/nw, c)) nw - h + 1,
//   result = sum_i x_i (v(c_{i+1}) - v(c_i))   (NaN without samples).
//
// One warp owns one (hour, cell) and sweeps its day axis with a sliding sorted
// window.  The padded day axis is indexed by P = d + tap (tap 0 .. 2h); position
// P holds day slot (P - h) mod n, so the wrap repeats slots when n < 2h + 1.
// Only the 2h - 1 nonzero-weight taps enter the sorted window: entries are
// (value, P) in shared memory, and an entry's weight is tri(P - d) = h - |P-d-h|
// (create_window_weights up to a scale, which the formula above cancels).
// Per output day:
//   1. sum w and sum w^2 from the per-position valid counts (O(window)),
//   2. one pass over the window: an integer warp scan of the weights gives every
//      entry's cumulative interval; only the 32-entry chunks whose interval meets
//      some quantile's [(h-1)/nw, h/nw] compute contributions.  The same pass
//      compacts out the entries of P = d + 1, which reach tap 0 on day d + 1,
//   3. merge in position P = d + 2h: its nitem samples, sorted by rank, are
//      placed by upper-bound search; the old entries move up from the back in
//      place (an entry only ever moves to a higher index).
// The results are accumulated as K + sum (x_i - K) dv_i with K the smallest
// value of the window, so a constant window returns its value exactly.
//
// SEEPS: samples below the dry threshold (compared in the series' precision)
// leave the sorted window like NaN, and the dry fraction is the UNWEIGHTED
// mean of x < threshold over all nyear * (2h + 1) samples, the zero-weight end
// taps and the NaN samples (never dry) included.  The dry counts slide per
// position like the valid counts.
//
// The samples of a position are read by the whole CTA at once (thread i reads
// cell i % cpb of year i / cpb), so a CTA of 8 float32 / 4 float64 cells reads
// whole 32-B sectors; the day-365 fill (utils.py:105) happens on load.
#include <math_constants.h>

#include <algorithm>

#include "climatology.cuh"

namespace wb2 {

constexpr int kQuantMaxQ = 16;            // quantiles per launch
constexpr int kQuantMaxSamples = 8192;    // nitem * window_size

struct QuantArgs {
  ClimArgs t;                  // tables; t.mean / t.std unused
  const double* q;             // [nq] quantiles
  const int32_t* hour_nyear;   // [nhour] stacked years of hour h
  int32_t nq, seeps;
  double dry;                  // dry threshold in the series' units (SEEPS)
  float* out;                  // [nhour][nq][nday_out][out_stride]
  float* dry_fraction;         // [nhour][nday_out][out_stride] (SEEPS)
  int32_t cap;                 // nitem * (window_size - 2) window entries
  int32_t stage_bytes, warp_bytes;
};

__device__ __forceinline__ int qwrap(int i, int n) {
  i %= n;
  return i < 0 ? i + n : i;
}

template <typename T>
__global__ void __launch_bounds__(256, 1) climatology_quantile_kernel(const T* __restrict__ x,
                                                                   QuantArgs a) {
  extern __shared__ __align__(16) unsigned char qsmem[];
  const unsigned full = 0xffffffffu;
  const int cpb = blockDim.x / 32;
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int h = blockIdx.y;
  const int64_t cell0 = int64_t(blockIdx.x) * cpb;
  const int64_t cell = cell0 + warp;
  const int n = a.t.hour_nday[h];
  const int nitem = a.t.nitem, hw = a.t.half, W = 2 * hw + 1;
  const int64_t* items = a.t.items + int64_t(h) * a.t.nday * nitem;
  const int64_t* fill = a.t.fill + int64_t(h) * nitem;
  const T thr = static_cast<T>(a.dry);
  const bool seeps = a.seeps != 0;

  T* stage = reinterpret_cast<T*>(qsmem);  // [cpb][nitem] raw samples of one position
  unsigned char* wb = qsmem + a.stage_bytes + size_t(warp) * a.warp_bytes;
  T* win_v = reinterpret_cast<T*>(wb);            // [cap] sorted window values
  T* bat = win_v + a.cap;                         // [nitem] sorted samples of one position
  double* qlo = reinterpret_cast<double*>(
      wb + ((size_t(a.cap) + nitem) * sizeof(T) + 7) / 8 * 8);  // [kQuantMaxQ]
  double* qhi = qlo + kQuantMaxQ;
  double* qh = qhi + kQuantMaxQ;
  double* acc = qh + kQuantMaxQ;
  int* win_p = reinterpret_cast<int*>(acc + kQuantMaxQ);  // [cap] position P of an entry
  int* ins = win_p + a.cap;                               // [nitem] merge ranks
  int* cnt = ins + nitem;                                 // [W] valid samples at P % W
  int* drc = cnt + W;                                     // [W] dry samples at P % W
  const T* mine = stage + warp * nitem;
  int m = 0, k = 0;  // entries in the window / in the batch

  auto usable = [&](T v) { return v == v && !(seeps && v < thr); };

  // samples of position P -> bat (sorted, NaN / dry dropped), counts at P % W.
  // Every thread of the CTA calls it (two barriers).
  auto load = [&](int P) {
    __syncthreads();  // the stage is free
    const int64_t* it = items + int64_t(qwrap(P - hw, n)) * nitem;
    for (int i = threadIdx.x; i < nitem * cpb; i += blockDim.x) {
      const int c = i % cpb, j = i / cpb;
      const int64_t cc = cell0 + c;
      T v = T(CUDART_NAN);
      if (cc < a.t.ncell) {
        const int64_t s = it[j];
        if (s >= 0) v = ldg_stream(x + s * a.t.tstride + cc);
        if (!(v == v)) {
          const int64_t f = fill[j];
          v = f >= 0 ? ldg_stream(x + f * a.t.tstride + cc) : T(CUDART_NAN);
        }
      }
      stage[c * nitem + j] = v;
    }
    __syncthreads();
    int nv = 0, nd = 0;
    for (int j = lane; j - lane < nitem; j += 32) {
      const T v = j < nitem ? mine[j] : T(CUDART_NAN);
      nv += __popc(__ballot_sync(full, j < nitem && usable(v)));
      nd += __popc(__ballot_sync(full, seeps && v < thr));
    }
    for (int j = lane; j < nitem; j += 32) {
      const T v = mine[j];
      if (!usable(v)) continue;
      int r = 0;
      for (int i = 0; i < nitem; ++i) {
        const T u = mine[i];
        r += usable(u) && (u < v || (u == v && i < j));
      }
      bat[r] = v;
    }
    if (lane == 0) {
      cnt[P % W] = nv;
      drc[P % W] = nd;
    }
    k = nv;
    __syncwarp();
  };

  // bat (k entries at position P) into the window
  auto merge = [&](int P) {
    for (int i = lane; i < k; i += 32) {
      const T b = bat[i];
      int lo = 0, hi = m;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (win_v[mid] <= b) lo = mid + 1;
        else hi = mid;
      }
      ins[i] = lo;
    }
    __syncwarp();
    if (k > 0)
      for (int base = (m - 1) & ~31; base >= 0 && m > 0; base -= 32) {
        const int e = base + lane;
        T v{};
        int p = 0, s = 0;
        if (e < m) {
          v = win_v[e];
          p = win_p[e];
          int lo = 0, hi = k;  // batch entries placed before entry e
          while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (ins[mid] <= e) lo = mid + 1;
            else hi = mid;
          }
          s = lo;
        }
        __syncwarp();
        if (e < m) {
          win_v[e + s] = v;
          win_p[e + s] = p;
        }
        __syncwarp();
      }
    for (int i = lane; i < k; i += 32) {
      win_v[ins[i] + i] = bat[i];
      win_p[ins[i] + i] = P;
    }
    m += k;
    __syncwarp();
  };

  for (int P = 0; P <= 2 * hw; ++P) {
    load(P);
    if (P >= 1 && P < 2 * hw) merge(P);
  }

  const int32_t* rows = a.t.out_row + int64_t(h) * a.t.nday;
  const double dry_den = double(a.hour_nyear[h]) * W;
  for (int d = 0; d < n; ++d) {
    // 1. sum w, sum w^2 over the nonzero taps; dry samples over all taps
    double s1 = 0.0, s2 = 0.0, nd = 0.0;
    for (int j = lane; j <= 2 * hw; j += 32) {
      const int r = (d + j) % W;
      const double w = double(hw - abs(j - hw));
      s1 = fma(w, double(cnt[r]), s1);
      s2 = fma(w * w, double(cnt[r]), s2);
      nd += double(drc[r]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s1 += __shfl_xor_sync(full, s1, o);
      s2 += __shfl_xor_sync(full, s2, o);
      nd += __shfl_xor_sync(full, nd, o);
    }
    const double nw = s2 > 0.0 ? s1 * s1 / s2 : 0.0;
    if (lane < a.nq) {
      const double hq = fmin(fmax((nw - 1.0) * a.q[lane] + 1.0, 1.0), nw);
      qh[lane] = hq;
      qlo[lane] = (hq - 1.0) / nw;
      qhi[lane] = hq / nw;
      acc[lane] = 0.0;
    }
    __syncwarp();
    const double K = m > 0 ? double(win_v[0]) : 0.0;

    // 2. weighted prefix pass; compacts out position d + 1
    int carry = 0, kept = 0;
    for (int base = 0; base < m; base += 32) {
      const int e = base + lane;
      T v{};
      int p = -1, w = 0;
      if (e < m) {
        v = win_v[e];
        p = win_p[e];
        w = hw - abs(p - d - hw);
      }
      int incl = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(full, incl, o);
        if (lane >= o) incl += y;
      }
      const int total = __shfl_sync(full, incl, 31);
      const double c_lo = double(carry) / s1, c_hi = double(carry + total) / s1;
      for (int qi = 0; qi < a.nq; ++qi) {
        if (!(c_hi > qlo[qi] && c_lo < qhi[qi])) continue;  // warp-uniform
        const double lo = qlo[qi], hi = qhi[qi], hq = qh[qi];
        const double cb = double(carry + incl - w) / s1, ca = double(carry + incl) / s1;
        const double vb = fmax(lo, fmin(hi, cb)) * nw - hq + 1.0;
        const double va = fmax(lo, fmin(hi, ca)) * nw - hq + 1.0;
        double c = e < m ? (double(v) - K) * (va - vb) : 0.0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(full, c, o);
        if (lane == 0) acc[qi] += c;
      }
      carry += total;
      const bool keep = e < m && p != d + 1;
      const unsigned bal = __ballot_sync(full, keep);
      const int pos = kept + __popc(bal & ((1u << lane) - 1u));
      __syncwarp();
      if (keep) {
        win_v[pos] = v;
        win_p[pos] = p;
      }
      kept += __popc(bal);
      __syncwarp();
    }
    if (cell < a.t.ncell && lane < a.nq) {
      const int64_t o =
          ((int64_t(h) * a.nq + lane) * a.t.nday_out + rows[d]) * a.t.out_stride + cell;
      a.out[o] = s1 > 0.0 ? static_cast<float>(K + acc[lane]) : CUDART_NAN_F;
    }
    if (cell < a.t.ncell && lane == 0 && a.dry_fraction)
      a.dry_fraction[(int64_t(h) * a.t.nday_out + rows[d]) * a.t.out_stride + cell] =
          static_cast<float>(nd / dry_den);
    m = kept;

    // 3. position d + 2h in, d + 2h + 1 loaded (counted now, merged tomorrow)
    if (d + 1 < n) {
      merge(d + 2 * hw);
      load(d + 2 * hw + 1);
    }
  }
}

// per-warp shared memory: window values + batch, the per-quantile scalars, then
// the int arrays (entry positions, merge ranks, the two count rings)
static size_t quant_warp_bytes(int cap, int nitem, int W, size_t esize) {
  const size_t v = ((size_t(cap) + nitem) * esize + 7) / 8 * 8;
  const size_t b = v + 4 * kQuantMaxQ * 8 + (size_t(cap) + nitem + 2 * size_t(W)) * 4;
  return (b + 15) / 16 * 16;
}

static int quant_launch(wb2_ctx* ctx, const void* x, int dtype, int64_t ncell,
                        const ClimArgs& t, QuantArgs q, float* out, float* dry_fraction) {
  q.t = t;
  q.t.ncell = ncell;
  q.t.tstride = ncell;
  q.t.out_stride = ncell;
  q.out = out;
  q.dry_fraction = dry_fraction;
  const size_t esize = dtype == WB2_F32 ? 4 : 8;
  const int W = 2 * t.half + 1;
  q.cap = t.nitem * (W - 2);
  const size_t warp_bytes = quant_warp_bytes(q.cap, t.nitem, W, esize);
  int max_smem = 0;
  WB2_CUDA_TRY(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin,
                                      ctx->device));
  // 8 cells per CTA (whole sectors of float32) when they fit, else fewer
  int cpb = dtype == WB2_F32 ? 8 : 4;
  auto smem_of = [&](int c) {
    return (size_t(c) * t.nitem * esize + 15) / 16 * 16 + size_t(c) * warp_bytes;
  };
  while (cpb > 1 && smem_of(cpb) > size_t(max_smem)) cpb /= 2;
  const size_t smem = smem_of(cpb);
  WB2_REQUIRE(smem <= size_t(max_smem), "one cell's window needs %zu B of shared memory", smem);
  q.stage_bytes = static_cast<int32_t>((size_t(cpb) * t.nitem * esize + 15) / 16 * 16);
  q.warp_bytes = static_cast<int32_t>(warp_bytes);
  const dim3 grid(static_cast<unsigned>((ncell + cpb - 1) / cpb),
                  static_cast<unsigned>(t.nhour));
  if (dtype == WB2_F32) {
    WB2_CUDA_TRY(cudaFuncSetAttribute(climatology_quantile_kernel<float>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
    climatology_quantile_kernel<float><<<grid, 32 * cpb, smem, ctx->stream>>>(
        static_cast<const float*>(x), q);
  } else {
    WB2_CUDA_TRY(cudaFuncSetAttribute(climatology_quantile_kernel<double>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
    climatology_quantile_kernel<double><<<grid, 32 * cpb, smem, ctx->stream>>>(
        static_cast<const double*>(x), q);
  }
  WB2_CUDA_TRY(cudaGetLastError());
  ctx->launches += 1;
  return WB2_OK;
}

// Checks shared by both entries; the quantiles and the per-hour year counts go
// to the device in one block.
static int quant_prepare(wb2_ctx* ctx, int dtype, int64_t ncell, int64_t nres, int32_t nhour,
                         int32_t nday, int32_t nitem, const int64_t* items,
                         const int32_t* hour_nday, int32_t window_size, int32_t nq,
                         const double* quantiles, int32_t seeps, double dry_threshold,
                         const float* dry_fraction, QuantArgs* q, DeviceBlock* blk) {
  WB2_REQUIRE(dtype == WB2_F32 || dtype == WB2_F64, "dtype must be WB2_F32 or WB2_F64");
  WB2_REQUIRE(nres == 0 || dtype == WB2_F32, "nres > 0 (the daily resample) takes float32 input");
  WB2_REQUIRE(ncell >= 0, "ncell < 0");
  WB2_REQUIRE(nq >= 1 && nq <= kQuantMaxQ, "nquantile must be in 1..%d (got %d)", kQuantMaxQ,
              nq);
  WB2_REQUIRE(quantiles != nullptr, "quantiles is NULL");
  for (int i = 0; i < nq; ++i)
    WB2_REQUIRE(quantiles[i] >= 0.0 && quantiles[i] <= 1.0,
                "quantiles[%d] = %g is outside [0, 1]", i, quantiles[i]);
  WB2_REQUIRE(seeps == 0 || seeps == 1, "seeps must be 0 or 1");
  WB2_REQUIRE(seeps == 0 || dry_fraction != nullptr, "SEEPS needs the dry_fraction output");
  WB2_REQUIRE(seeps == 1 || dry_fraction == nullptr, "dry_fraction is a SEEPS output");
  WB2_REQUIRE(int64_t(nitem) * window_size <= kQuantMaxSamples,
              "nitem * window_size = %lld exceeds %d samples per window",
              static_cast<long long>(int64_t(nitem) * window_size), kQuantMaxSamples);
  *q = QuantArgs{};
  q->nq = nq;
  q->seeps = seeps;
  q->dry = dry_threshold;
  // stacked years of each hour: the item columns that hold any step
  std::vector<int32_t> ny(size_t(nhour), 0);
  for (int32_t h = 0; h < nhour; ++h)
    for (int32_t j = 0; j < nitem; ++j)
      for (int32_t d = 0; d < hour_nday[h]; ++d)
        if (items[(int64_t(h) * nday + d) * nitem + j] >= 0) {
          ny[size_t(h)] += 1;
          break;
        }
  if (ncell == 0) return WB2_OK;
  size_t o[2];
  WB2_TRY(upload_parts(ctx, {{quantiles, size_t(nq) * 8}, {ny.data(), ny.size() * 4}}, blk, o));
  q->q = blk->at<const double>(o[0]);
  q->hour_nyear = blk->at<const int32_t>(o[1]);
  return WB2_OK;
}

}  // namespace wb2

using namespace wb2;

extern "C" {

int wb2_climatology_quantile(wb2_ctx* ctx, const void* x, int dtype, int64_t ntime,
                             int64_t ncell, int64_t nres, const int64_t* res_start,
                             const int32_t* res_count, int32_t nhour, int32_t nday,
                             int32_t nitem, const int64_t* items, const int64_t* fill,
                             const int32_t* hour_nday, const int32_t* out_row, int32_t nday_out,
                             int32_t window_size, int32_t nquantile, const double* quantiles,
                             int32_t seeps, double dry_threshold, float* out,
                             float* dry_fraction) {
  WB2_NVTX("wb2_climatology_quantile");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  ClimPlan p;
  WB2_TRY(clim_validate(ntime, nres, res_start, res_count, nhour, nday, nitem, items, fill,
                        hour_nday, out_row, nday_out, window_size, 0, &p));
  WB2_REQUIRE(out != nullptr || ncell == 0, "out is NULL");
  DeviceGuard guard(ctx->device);
  QuantArgs q;
  DeviceBlock nyear, tables, daily;
  WB2_TRY(quant_prepare(ctx, dtype, ncell, nres, nhour, nday, nitem, items, hour_nday,
                        window_size, nquantile, quantiles, seeps, dry_threshold, dry_fraction, &q,
                        &nyear));
  if (ncell == 0) return WB2_OK;
  WB2_REQUIRE(x != nullptr, "x is NULL");
  ClimArgs args;
  WB2_TRY(clim_upload(ctx, p, items, p.fill, &tables, &args));
  const void* src = x;
  if (nres > 0) {
    WB2_TRY(daily.alloc(ctx, size_t(nres) * ncell * 4));
    WB2_TRY(clim_resample(ctx, static_cast<const float*>(x), ncell, ncell, p, res_start,
                          daily.at<float>(0)));
    src = daily.at<float>(0);
  }
  if (p.need_nan_fill) {  // day labels some hour does not have
    const size_t rows = size_t(nhour) * nday_out * ncell * 4;
    WB2_CUDA_TRY(cudaMemsetAsync(out, 0xFF, rows * nquantile, ctx->stream));
    if (dry_fraction) WB2_CUDA_TRY(cudaMemsetAsync(dry_fraction, 0xFF, rows, ctx->stream));
  }
  return quant_launch(ctx, src, dtype, ncell, args, q, out, dry_fraction);
}

int wb2_climatology_quantile_host(wb2_ctx* ctx, const void* x, int dtype, int64_t ntime,
                                  int64_t ncell, int64_t nres, const int64_t* res_start,
                                  const int32_t* res_count, int32_t nhour, int32_t nday,
                                  int32_t nitem, const int64_t* items, const int64_t* fill,
                                  const int32_t* hour_nday, const int32_t* out_row,
                                  int32_t nday_out, int32_t window_size, int32_t nquantile,
                                  const double* quantiles, int32_t seeps,
                                  double dry_threshold, size_t budget, float* out_host,
                                  float* dry_fraction_host) {
  WB2_NVTX("wb2_climatology_quantile_host");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  ClimPlan p;
  WB2_TRY(clim_validate(ntime, nres, res_start, res_count, nhour, nday, nitem, items, fill,
                        hour_nday, out_row, nday_out, window_size, 0, &p));
  WB2_REQUIRE(out_host != nullptr || ncell == 0, "out is NULL");
  DeviceGuard guard(ctx->device);
  QuantArgs q;
  DeviceBlock nyear;
  WB2_TRY(quant_prepare(ctx, dtype, ncell, nres, nhour, nday, nitem, items, hour_nday,
                        window_size, nquantile, quantiles, seeps, dry_threshold,
                        dry_fraction_host, &q, &nyear));
  if (ncell == 0) return WB2_OK;
  WB2_REQUIRE(x != nullptr, "x is NULL");
  float* const out[2] = {out_host, dry_fraction_host};
  const size_t rows = size_t(nhour) * nday_out;
  const size_t out_rows[2] = {rows * nquantile, rows};
  return clim_stream_host(
      ctx, x, dtype, ntime, ncell, p, budget, seeps ? 2 : 1, out, out_rows,
      [&](const void* src, int64_t n, const ClimArgs& tables, float* const* o) {
        return quant_launch(ctx, src, dtype, n, tables, q, o[0], seeps ? o[1] : nullptr);
      });
}

}  // extern "C"

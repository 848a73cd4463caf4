// Day-of-year climatologies: wb2_climatology (device-resident series) and
// wb2_climatology_host (NumPy / memmap series streamed in bands of cells).
//
// Replaces compute_rolling_stat / compute_hourly_stat / compute_daily_stat and
// their `_fast` variants (weatherbench2/utils.py:88-287), the hot path of
// scripts/compute_climatology.py.  The host turns the time selection into an
// index table -- for every (hour, day slot) the time steps that feed it (one per
// stacked year for the explicit method, every step with that day-of-year label
// for the fast method), -1 for a missing slot -- and the kernel reads the
// (time, cells) series in place through it.
//
// One CTA owns 8 cells (one 32-B sector of float32 per time step) and the whole
// day axis of one hour:
//   phase 1  per (day slot, cell) the float64 moments over the slot's items:
//            count, sum (x - K), sum (x - K)^2, K = a per-cell shift (a
//            finite value of the cell, found by probing up to 512 table
//            entries spread over the whole table) so that fields with a
//            large mean keep their variance, even when the first entries of
//            the table are missing or NaN.  The explicit method fills a NaN /
//            missing item of year y with year y's day-365 value on load
//            (utils.py:105).  The moments live in shared memory (20 B per day
//            and cell: 58.5 KB for 366 days), never in HBM.
//   phase 2  the circular 2h+1-tap triangular window over the positional day
//            axis.  Triangle = box * box, so every weighted sum slides with
//            three running sums (T += R - L; R and L are the right / left
//            half boxes): O(1) work per output day instead of O(2h+1).
//              explicit: mean = K + T1/T0, std = sqrt(T2/T0 - (T1/T0)^2)
//                        (xarray's weighted mean / population std over
//                        (window, year), NaN where the weight sum is 0)
//              fast:     per-day groupby mean / std (ddof 0) first, then
//                        mean over the 2h+1 taps of w * value, NaN skipped,
//                        divided by the COUNT of valid taps (utils.py:169-197)
// Mean and std come out of the same read of the input.
//
// The daily `resample(time='D').mean()` of the daily statistics is
// wb2_ens_mean over consecutive time slabs (member_stride = time stride).
#include <math_constants.h>

#include <algorithm>

#include "climatology.cuh"

namespace wb2 {

constexpr int kClimCells = 8;   // cells per CTA
constexpr int kClimLanes = 32;  // day lanes per CTA
constexpr int kClimThreads = kClimCells * kClimLanes;
constexpr int kClimMaxDays = 1400;  // shared memory: 160 B per day slot
constexpr int kClimShiftSamples = 512;  // table entries probed for the shift

__device__ __forceinline__ int wrap_day(int i, int n) {
  i %= n;
  return i < 0 ? i + n : i;
}

template <typename T>
__global__ void __launch_bounds__(kClimThreads) climatology_kernel(const T* __restrict__ x,
                                                                   ClimArgs a) {
  extern __shared__ double clim_smem[];
  __shared__ double shift[kClimCells];
  __shared__ int first[kClimCells];
  double* s1 = clim_smem;                 // [nday][8]
  double* s2 = s1 + a.nday * kClimCells;  // [nday][8]
  float* cnt = reinterpret_cast<float*>(s2 + a.nday * kClimCells);
  const int cl = threadIdx.x % kClimCells, dl = threadIdx.x / kClimCells;
  const int h = blockIdx.y;
  const int64_t cell = int64_t(blockIdx.x) * kClimCells + cl;
  const bool live = cell < a.ncell;
  const int n = a.hour_nday[h];
  const int nitem = a.nitem;
  const int64_t* items = a.items + int64_t(h) * a.nday * nitem;
  const int64_t* fill = a.fill ? a.fill + int64_t(h) * nitem : nullptr;
  const T* xc = x + (live ? cell : 0);

  // The shift K: the cell's value at the first of kClimShiftSamples table
  // entries, spread evenly over the hour's whole table (every entry when it
  // has fewer), that is finite after the fill.  Day lane 0 probes entry 0,
  // which settles almost every cell with one load; otherwise the 32 day lanes
  // of the cell probe in parallel, so a cell that is NaN everywhere costs
  // each lane kClimShiftSamples / 32 probes.  K = 0 only when no probe is
  // finite.
  const int64_t nentry = int64_t(n) * nitem;
  const int nprobe = nentry < kClimShiftSamples ? int(nentry) : kClimShiftSamples;
  auto probe = [&](int i) {  // the value at entry i of the nprobe, fill applied
    const int64_t q = nprobe == nentry ? i : int64_t(i) * nentry / nprobe;
    const int64_t t = items[q];
    double v = t >= 0 ? double(ldg_stream(xc + t * a.tstride)) : CUDART_NAN;
    if (fill != nullptr && !(v == v)) {
      const int64_t f = fill[q % nitem];
      v = f >= 0 ? double(ldg_stream(xc + f * a.tstride)) : CUDART_NAN;
    }
    return v;
  };
  if (dl == 0) {
    const double v = live ? probe(0) : CUDART_NAN;
    shift[cl] = v == v ? v : 0.0;
    first[cl] = v == v ? 0 : kClimShiftSamples;
  }
  __syncthreads();
  int hit = kClimShiftSamples;
  double hv = 0.0;
  if (first[cl] != 0)
    for (int i = dl; live && i < nprobe; i += kClimLanes) {
      const double v = probe(i);
      if (v == v) {
        hit = i;
        hv = v;
        atomicMin(&first[cl], i);
        break;
      }
    }
  __syncthreads();
  if (hit < kClimShiftSamples && hit == first[cl]) shift[cl] = hv;  // one lane
  __syncthreads();
  const double k = shift[cl];

  // phase 1: per-slot moments (years of a slot in flight together)
  for (int d = dl; d < n; d += kClimLanes) {
    double m1 = 0.0, m2 = 0.0;
    float c = 0.f;
    const int64_t* it = items + int64_t(d) * nitem;
    if (live) {
#pragma unroll 4
      for (int j = 0; j < nitem; ++j) {
        const int64_t t = it[j];
        double v = t >= 0 ? double(ldg_stream(xc + t * a.tstride)) : CUDART_NAN;
        if (fill != nullptr && !(v == v)) {
          const int64_t f = fill[j];
          v = f >= 0 ? double(ldg_stream(xc + f * a.tstride)) : CUDART_NAN;
        }
        if (v == v) {
          v -= k;
          m1 += v;
          m2 = fma(v, v, m2);
          c += 1.f;
        }
      }
    }
    s1[d * kClimCells + cl] = m1;
    s2[d * kClimCells + cl] = m2;
    cnt[d * kClimCells + cl] = c;
  }
  __syncthreads();
  if (a.fast) {  // groupby mean / std (ddof 0) per day; cnt becomes "value valid"
    for (int d = dl; d < n; d += kClimLanes) {
      const int i = d * kClimCells + cl;
      const double c = cnt[i];
      if (c > 0.0) {
        const double mu = s1[i] / c;
        s1[i] = mu;
        s2[i] = sqrt(fmax(s2[i] / c - mu * mu, 0.0));
        cnt[i] = 1.f;
      } else {
        s1[i] = s2[i] = 0.0;
        cnt[i] = 0.f;
      }
    }
    __syncthreads();
  }

  // phase 2: sliding triangular window over a run of consecutive days
  const int chunk = (n + kClimLanes - 1) / kClimLanes;
  const int d0 = dl * chunk, d1 = min(n, d0 + chunk);
  if (!live || d0 >= d1) return;
  const int hw = a.half;
  double tri[3] = {0.0, 0.0, 0.0}, rb[3] = {0.0, 0.0, 0.0}, lb[3] = {0.0, 0.0, 0.0};
  double box = 0.0;
  for (int j = -hw; j <= hw; ++j) {
    const int i = wrap_day(d0 + j, n) * kClimCells + cl;
    const double v[3] = {double(cnt[i]), s1[i], s2[i]};
    const double wt = double(hw - abs(j));
    box += v[0];
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      tri[q] = fma(wt, v[q], tri[q]);
      if (j >= 1) rb[q] += v[q];
      else if (j > -hw) lb[q] += v[q];
    }
  }
  const double fast_scale = double(2 * hw + 1) / (double(hw) * double(hw));
  const int32_t* rows = a.out_row + int64_t(h) * a.nday;
  for (int d = d0; d < d1; ++d) {
    float mv = CUDART_NAN_F, sv = CUDART_NAN_F;
    if (!a.fast) {
      if (tri[0] > 0.0) {
        const double mu = tri[1] / tri[0];
        mv = static_cast<float>(k + mu);
        sv = static_cast<float>(sqrt(fmax(tri[2] / tri[0] - mu * mu, 0.0)));
      }
    } else if (box > 0.0) {
      mv = static_cast<float>(fast_scale * fma(k, tri[0], tri[1]) / box);
      sv = static_cast<float>(fast_scale * tri[2] / box);
    }
    const int64_t o = (int64_t(h) * a.nday_out + rows[d]) * a.out_stride + cell;
    if (a.mean) a.mean[o] = mv;
    if (a.std) a.std[o] = sv;
    if (d + 1 == d1) break;
    const int ip = wrap_day(d + hw + 1, n) * kClimCells + cl;
    const int i1 = wrap_day(d + 1, n) * kClimCells + cl;
    const int im = wrap_day(d - hw + 1, n) * kClimCells + cl;
    const int ib = wrap_day(d - hw, n) * kClimCells + cl;
    const double vp[3] = {double(cnt[ip]), s1[ip], s2[ip]};
    const double v1[3] = {double(cnt[i1]), s1[i1], s2[i1]};
    const double vm[3] = {double(cnt[im]), s1[im], s2[im]};
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      tri[q] += rb[q] - lb[q];
      rb[q] += vp[q] - v1[q];
      lb[q] += v1[q] - vm[q];
    }
    box += double(cnt[ip]) - double(cnt[ib]);
  }
}

int clim_validate(int64_t ntime, int64_t nres, const int64_t* res_start,
                         const int32_t* res_count, int32_t nhour, int32_t nday, int32_t nitem,
                         const int64_t* items, const int64_t* fill, const int32_t* hour_nday,
                         const int32_t* out_row, int32_t nday_out, int32_t window_size,
                         int32_t method, ClimPlan* p) {
  WB2_REQUIRE(window_size >= 3 && window_size % 2 == 1,
              "window_size must be odd and >= 3 (got %d)", window_size);
  WB2_REQUIRE(method == 0 || method == 1, "method must be 0 (explicit) or 1 (fast)");
  WB2_REQUIRE(nhour >= 1 && nhour <= 65535, "nhour must be in 1..65535 (got %d)", nhour);
  WB2_REQUIRE(nday >= 1 && nday <= kClimMaxDays, "nday must be in 1..%d (got %d)",
              kClimMaxDays, nday);
  WB2_REQUIRE(nitem >= 1 && nday_out >= 1, "nitem and nday_out must be >= 1");
  WB2_REQUIRE(ntime >= 0 && nres >= 0, "ntime / nres must be >= 0");
  WB2_REQUIRE(items && hour_nday && out_row, "items / hour_nday / out_row are NULL");
  WB2_REQUIRE(method == 1 || fill != nullptr, "the explicit method needs the fill table");
  if (nres > 0) WB2_REQUIRE(res_start && res_count, "res_start / res_count are NULL");
  // steps the table refers to: resampled days, or raw time steps
  const int64_t nsrc = nres > 0 ? nres : ntime;
  for (int64_t i = 0; i < nres; ++i) {
    WB2_REQUIRE(res_count[i] >= 0 && res_count[i] <= ntime, "bad res_count[%lld]",
                static_cast<long long>(i));
    if (res_count[i] > 0)
      WB2_REQUIRE(res_start[i] >= 0 && res_start[i] + res_count[i] <= ntime,
                  "res_start[%lld] out of range", static_cast<long long>(i));
  }
  p->need_nan_fill = false;
  std::vector<int32_t> row_owner(size_t(nday_out), -1);  // hour that wrote the row
  for (int32_t h = 0; h < nhour; ++h) {
    const int32_t n = hour_nday[h];
    WB2_REQUIRE(n >= 1 && n <= nday, "hour_nday[%d] = %d out of 1..%d", h, n, nday);
    if (n < nday_out) p->need_nan_fill = true;
    for (int32_t d = 0; d < n; ++d) {
      const int32_t r = out_row[int64_t(h) * nday + d];
      WB2_REQUIRE(r >= 0 && r < nday_out, "out_row[%d][%d] = %d out of range", h, d, r);
      WB2_REQUIRE(row_owner[size_t(r)] != h,
                  "out_row[%d][%d] = %d repeats a row of hour %d (rows must be distinct)",
                  h, d, r, h);
      row_owner[size_t(r)] = h;
      for (int32_t j = 0; j < nitem; ++j) {
        const int64_t t = items[(int64_t(h) * nday + d) * nitem + j];
        WB2_REQUIRE(t >= -1 && t < nsrc, "items[%d][%d][%d] = %lld out of range", h, d, j,
                    static_cast<long long>(t));
      }
    }
    if (fill)
      for (int32_t j = 0; j < nitem; ++j) {
        const int64_t t = fill[int64_t(h) * nitem + j];
        WB2_REQUIRE(t >= -1 && t < nsrc, "fill[%d][%d] out of range", h, j);
      }
  }
  p->nres = nres;
  p->res_start = res_start;
  p->res_count = res_count;
  p->nhour = nhour;
  p->nday = nday;
  p->nitem = nitem;
  p->nday_out = nday_out;
  p->half = window_size / 2;
  p->fast = method;
  p->items = items;
  p->fill = method == 0 ? fill : nullptr;
  p->hour_nday = hour_nday;
  p->out_row = out_row;
  return WB2_OK;
}

int clim_upload(wb2_ctx* ctx, const ClimPlan& p, const int64_t* items, const int64_t* fill,
                DeviceBlock* blk, ClimArgs* a) {
  const size_t n_fill = p.fill ? size_t(p.nhour) * p.nitem : 0;
  size_t o[4];
  WB2_TRY(upload_parts(ctx,
                       {{items, size_t(p.nhour) * p.nday * p.nitem * 8},
                        {fill, n_fill * 8},
                        {p.hour_nday, size_t(p.nhour) * 4},
                        {p.out_row, size_t(p.nhour) * p.nday * 4}},
                       blk, o));
  *a = ClimArgs{};
  a->items = blk->at<const int64_t>(o[0]);
  a->fill = n_fill ? blk->at<const int64_t>(o[1]) : nullptr;
  a->hour_nday = blk->at<const int32_t>(o[2]);
  a->out_row = blk->at<const int32_t>(o[3]);
  a->nhour = p.nhour;
  a->nday = p.nday;
  a->nitem = p.nitem;
  a->nday_out = p.nday_out;
  a->half = p.half;
  a->fast = p.fast;
  return WB2_OK;
}

// resample(time='D').mean(): day i is the skip-NaN mean of `count[i]`
// consecutive time slabs from `start[i]` (NaN for a day without data).
int clim_resample(wb2_ctx* ctx, const float* x, int64_t tstride, int64_t ncell,
                  const ClimPlan& p, const int64_t* start, float* daily) {
  int64_t i = 0;
  std::vector<int64_t> off;
  while (i < p.nres) {
    const int32_t c = p.res_count[i];
    int64_t j = i + 1;
    while (j < p.nres && p.res_count[j] == c && j - i < 65535) ++j;
    if (c == 0) {
      WB2_CUDA_TRY(cudaMemsetAsync(daily + i * ncell, 0xFF, size_t(j - i) * ncell * 4,
                                   ctx->stream));
    } else {
      off.resize(size_t(j - i));
      for (int64_t q = i; q < j; ++q) off[size_t(q - i)] = start[q] * tstride;
      WB2_TRY(wb2_ens_mean(ctx, x, c, tstride, j - i, off.data(), ncell, 1,
                           daily + i * ncell));
    }
    i = j;
  }
  return WB2_OK;
}

static int clim_launch(wb2_ctx* ctx, const void* x, int dtype, int64_t ncell, int64_t tstride,
                       ClimArgs a, float* mean, float* std) {
  a.ncell = ncell;
  a.tstride = tstride;
  a.out_stride = ncell;
  a.mean = mean;
  a.std = std;
  const size_t smem = size_t(a.nday) * kClimCells * (8 + 8 + 4);
  const dim3 grid(static_cast<unsigned>((ncell + kClimCells - 1) / kClimCells),
                  static_cast<unsigned>(a.nhour));
  if (dtype == WB2_F32) {
    WB2_CUDA_TRY(cudaFuncSetAttribute(climatology_kernel<float>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
    climatology_kernel<float><<<grid, kClimThreads, smem, ctx->stream>>>(
        static_cast<const float*>(x), a);
  } else {
    WB2_CUDA_TRY(cudaFuncSetAttribute(climatology_kernel<double>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
    climatology_kernel<double><<<grid, kClimThreads, smem, ctx->stream>>>(
        static_cast<const double*>(x), a);
  }
  WB2_CUDA_TRY(cudaGetLastError());
  ctx->launches += 1;
  return WB2_OK;
}

int clim_stream_host(wb2_ctx* ctx, const void* x, int dtype, int64_t ntime, int64_t ncell,
                     const ClimPlan& p, size_t budget, int nout, float* const* out_host,
                     const size_t* out_rows, const ClimBandFn& band) {
  const size_t esize = dtype == WB2_F32 ? 4 : 8;
  const int32_t nhour = p.nhour, nday = p.nday, nitem = p.nitem;
  const int64_t nres = p.nres;
  const int64_t* res_start = p.res_start;
  const int32_t* res_count = p.res_count;
  const int64_t* items = p.items;

  // the time rows the selection touches; tables rebased to the first of them
  int64_t t_lo = ntime, t_hi = -1;
  const size_t n_items = size_t(nhour) * nday * nitem;
  const size_t n_fill = p.fill ? size_t(nhour) * nitem : 0;
  if (nres > 0) {
    for (int64_t i = 0; i < nres; ++i)
      if (res_count[i] > 0) {
        t_lo = std::min(t_lo, res_start[i]);
        t_hi = std::max(t_hi, res_start[i] + res_count[i] - 1);
      }
  } else {
    for (size_t i = 0; i < n_items; ++i)
      if (items[i] >= 0) t_lo = std::min(t_lo, items[i]), t_hi = std::max(t_hi, items[i]);
    for (size_t i = 0; i < n_fill; ++i)
      if (p.fill[i] >= 0) t_lo = std::min(t_lo, p.fill[i]), t_hi = std::max(t_hi, p.fill[i]);
  }
  const int64_t rows = t_hi >= t_lo ? t_hi - t_lo + 1 : 0;
  if (rows == 0) t_lo = 0;
  std::vector<int64_t> it_r(items, items + n_items), fill_r, start_r;
  if (nres > 0) {
    start_r.assign(res_start, res_start + nres);
    for (auto& v : start_r) v -= t_lo;
  } else {
    for (auto& v : it_r)
      if (v >= 0) v -= t_lo;
  }
  if (n_fill) {
    fill_r.assign(p.fill, p.fill + n_fill);
    if (nres == 0)
      for (auto& v : fill_r)
        if (v >= 0) v -= t_lo;
  }

  // band of cells: input rows + resampled days + outputs, double buffered
  size_t out_per_cell = 0;
  for (int s = 0; s < nout; ++s) out_per_cell += out_rows[s] * 4;
  const size_t per_cell = size_t(rows) * esize + size_t(nres) * 4 + out_per_cell;
  int64_t nb = static_cast<int64_t>(budget / (2 * per_cell));
  nb = std::max<int64_t>(1, std::min(nb, ncell));
  auto al = [](size_t b) { return (b + 255) / 256 * 256; };
  const size_t b_in = al(size_t(rows) * nb * esize), b_day = al(size_t(nres) * nb * 4);
  std::vector<size_t> b_out(static_cast<size_t>(nout));
  size_t stage_bytes = b_in + b_day;
  for (int s = 0; s < nout; ++s) stage_bytes += b_out[size_t(s)] = al(out_rows[s] * nb * 4);

  DeviceBlock tables;
  ClimArgs args;
  WB2_TRY(clim_upload(ctx, p, it_r.data(), n_fill ? fill_r.data() : nullptr, &tables, &args));
  StagePair stage;
  WB2_TRY(stage.alloc(stage_bytes));
  StagePipe pipe(ctx, stage.buf[0], stage.buf[1]);
  const char* xh = static_cast<const char*>(x);
  std::vector<float*> out(static_cast<size_t>(nout));
  for (int64_t c0 = 0; c0 < ncell; c0 += nb) {
    const int64_t n = std::min(nb, ncell - c0);
    char* in;
    WB2_TRY(pipe.next(&in));
    float* daily = reinterpret_cast<float*>(in + b_in);
    char* o = in + b_in + b_day;
    for (int s = 0; s < nout; ++s) {
      out[size_t(s)] = reinterpret_cast<float*>(o);
      o += b_out[size_t(s)];
    }
    if (rows > 0)  // the band's whole selected series: one strided 2-D copy
      WB2_TRY(pipe.h2d_2d(in, size_t(n) * esize, xh + (size_t(t_lo) * ncell + c0) * esize,
                          size_t(ncell) * esize, size_t(n) * esize, size_t(rows)));
    WB2_TRY(pipe.ready());
    const void* src = in;
    if (nres > 0) {
      WB2_TRY(clim_resample(ctx, reinterpret_cast<const float*>(in), n, n, p, start_r.data(),
                            daily));
      src = daily;
    }
    if (p.need_nan_fill)
      WB2_CUDA_TRY(cudaMemsetAsync(out[0], 0xFF, size_t(o - reinterpret_cast<char*>(out[0])),
                                   ctx->stream));
    WB2_TRY(band(src, n, args, out.data()));
    for (int s = 0; s < nout; ++s)
      WB2_TRY(pipe.d2h_2d(out_host[s] + c0, size_t(ncell) * 4, out[size_t(s)], size_t(n) * 4,
                          size_t(n) * 4, out_rows[s]));
    WB2_TRY(pipe.done());
  }
  return pipe.finish();
}

}  // namespace wb2

using namespace wb2;

extern "C" {

int wb2_climatology(wb2_ctx* ctx, const void* x, int dtype, int64_t ntime, int64_t ncell,
                    int64_t nres, const int64_t* res_start, const int32_t* res_count,
                    int32_t nhour, int32_t nday, int32_t nitem, const int64_t* items,
                    const int64_t* fill, const int32_t* hour_nday, const int32_t* out_row,
                    int32_t nday_out, int32_t window_size, int32_t method, float* mean,
                    float* std) {
  WB2_NVTX("wb2_climatology");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_REQUIRE(dtype == WB2_F32 || dtype == WB2_F64, "dtype must be WB2_F32 or WB2_F64");
  WB2_REQUIRE(nres == 0 || dtype == WB2_F32, "nres > 0 (the daily resample) takes float32 input");
  WB2_REQUIRE(ncell >= 0, "ncell < 0");
  WB2_REQUIRE(mean || std, "neither mean nor std requested");
  ClimPlan p;
  WB2_TRY(clim_validate(ntime, nres, res_start, res_count, nhour, nday, nitem, items, fill,
                        hour_nday, out_row, nday_out, window_size, method, &p));
  if (ncell == 0) return WB2_OK;
  WB2_REQUIRE(x != nullptr, "x is NULL");
  DeviceGuard guard(ctx->device);
  DeviceBlock tables, daily;
  ClimArgs args;
  WB2_TRY(clim_upload(ctx, p, items, p.fill, &tables, &args));
  const void* src = x;
  if (nres > 0) {
    WB2_TRY(daily.alloc(ctx, size_t(nres) * ncell * 4));
    WB2_TRY(clim_resample(ctx, static_cast<const float*>(x), ncell, ncell, p, res_start,
                          daily.at<float>(0)));
    src = daily.at<float>(0);
  }
  const size_t out_bytes = size_t(nhour) * nday_out * ncell * 4;
  if (p.need_nan_fill) {  // day labels some hour does not have
    if (mean) WB2_CUDA_TRY(cudaMemsetAsync(mean, 0xFF, out_bytes, ctx->stream));
    if (std) WB2_CUDA_TRY(cudaMemsetAsync(std, 0xFF, out_bytes, ctx->stream));
  }
  return clim_launch(ctx, src, dtype, ncell, ncell, args, mean, std);
}

int wb2_climatology_host(wb2_ctx* ctx, const void* x, int dtype, int64_t ntime, int64_t ncell,
                         int64_t nres, const int64_t* res_start, const int32_t* res_count,
                         int32_t nhour, int32_t nday, int32_t nitem, const int64_t* items,
                         const int64_t* fill, const int32_t* hour_nday, const int32_t* out_row,
                         int32_t nday_out, int32_t window_size, int32_t method,
                         size_t budget, float* mean_host, float* std_host) {
  WB2_NVTX("wb2_climatology_host");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_REQUIRE(dtype == WB2_F32 || dtype == WB2_F64, "dtype must be WB2_F32 or WB2_F64");
  WB2_REQUIRE(nres == 0 || dtype == WB2_F32, "nres > 0 (the daily resample) takes float32 input");
  WB2_REQUIRE(ncell >= 0, "ncell < 0");
  WB2_REQUIRE(mean_host || std_host, "neither mean nor std requested");
  ClimPlan p;
  WB2_TRY(clim_validate(ntime, nres, res_start, res_count, nhour, nday, nitem, items, fill,
                        hour_nday, out_row, nday_out, window_size, method, &p));
  if (ncell == 0) return WB2_OK;
  WB2_REQUIRE(x != nullptr, "x is NULL");
  DeviceGuard guard(ctx->device);
  float* const out_host[2] = {mean_host ? mean_host : std_host, std_host};
  const size_t rows = size_t(nhour) * nday_out;
  const size_t out_rows[2] = {rows, rows};
  const int nout = (mean_host ? 1 : 0) + (std_host ? 1 : 0);
  return clim_stream_host(
      ctx, x, dtype, ntime, ncell, p, budget, nout, out_host, out_rows,
      [&](const void* src, int64_t n, const ClimArgs& tables, float* const* out) {
        return clim_launch(ctx, src, dtype, n, n, tables, mean_host ? out[0] : nullptr,
                           std_host ? out[nout - 1] : nullptr);
      });
}

}  // extern "C"

// Shared host side of the day-of-year climatology entries (climatology.cu and
// climatology_quantile.cu): the validated index tables, their device copy, the
// daily resample and the band loop that streams a host series through a
// StagePipe (stage.cuh).
#pragma once

#include <functional>

#include "stage.cuh"

namespace wb2 {

struct ClimArgs {
  const int64_t* items;      // [nhour][nday][nitem] time step (of the read series) or -1
  const int64_t* fill;       // [nhour][nitem] day-365 step of stacked year j, or NULL
  const int32_t* hour_nday;  // [nhour] day slots of this hour (the wrap period)
  const int32_t* out_row;    // [nhour][nday] output row of each day slot
  int64_t ncell;             // cells of this launch
  int64_t tstride;           // elements between consecutive time steps
  int64_t out_stride;        // elements between output rows
  int32_t nhour, nday, nitem, nday_out, half;
  int32_t fast;
  float* mean;  // [nhour][nday_out][out_stride] or NULL
  float* std;
};

// The caller's tables, validated.
struct ClimPlan {
  int64_t nres = 0;
  const int64_t* res_start = nullptr;  // host
  const int32_t* res_count = nullptr;  // host
  int32_t nhour = 0, nday = 0, nitem = 0, nday_out = 0, half = 0, fast = 0;
  const int64_t* items = nullptr;  // host
  const int64_t* fill = nullptr;
  const int32_t* hour_nday = nullptr;
  const int32_t* out_row = nullptr;
  bool need_nan_fill = false;  // some hour lacks some output day
};

int clim_validate(int64_t ntime, int64_t nres, const int64_t* res_start,
                  const int32_t* res_count, int32_t nhour, int32_t nday, int32_t nitem,
                  const int64_t* items, const int64_t* fill, const int32_t* hour_nday,
                  const int32_t* out_row, int32_t nday_out, int32_t window_size,
                  int32_t method, ClimPlan* p);

// Device copy of the tables, [items][fill][hour_nday][out_row] in `blk`; `a`
// gets their device pointers and the plan's sizes.
int clim_upload(wb2_ctx* ctx, const ClimPlan& p, const int64_t* items, const int64_t* fill,
                DeviceBlock* blk, ClimArgs* a);

// resample(time='D').mean() of a device series into `daily` [nres][ncell].
int clim_resample(wb2_ctx* ctx, const float* x, int64_t tstride, int64_t ncell,
                  const ClimPlan& p, const int64_t* start, float* daily);

// One band of `n` cells staged on the device: `src` is the band's series
// ([time][n], the resampled days when the plan resamples), `out[s]` the band's
// device output s ([out_rows[s]][n] float32), NaN-filled when some hour lacks
// an output day.  Enqueues the band's kernels on ctx->stream.
using ClimBandFn =
    std::function<int(const void* src, int64_t n, const ClimArgs& tables, float* const* out)>;

// The band loop of the *_host entries: bands of cells sized so that a private
// StagePair (selected input rows, resampled days and `nout` outputs of
// out_rows[s] rows each) fits `budget`; through a StagePipe, one strided 2-D
// copy per band overlaps the previous band's kernels; every output band is
// copied back into out_host[s] ([out_rows[s]][ncell]).
int clim_stream_host(wb2_ctx* ctx, const void* x, int dtype, int64_t ntime, int64_t ncell,
                     const ClimPlan& p, size_t budget, int nout, float* const* out_host,
                     const size_t* out_rows, const ClimBandFn& band);

}  // namespace wb2

// End-to-end entries for HOST-resident inputs (the *_host functions of
// include/wb2b200.h) and the device-resident slab cache behind them.
//
// The reference evaluates NumPy-backed xarray chunks
// (weatherbench2/evaluation.py:583-599, 693-705): every chunk materialises
// `truth.sel(time=valid_time)` (evaluation.py:475) and the climatology gather
// (metrics.py:398-404).  Here the 2-D slabs of a chunk are streamed through two
// device staging buffers -- H2D on a copy stream, overlapped with the kernel of
// the previous group and, for the entries that produce arrays, with the D2H of
// its result -- and the operands that repeat from chunk to chunk (truth and
// climatology slabs: consecutive init times share all but one valid time) can
// be kept in an LRU SLAB CACHE in HBM, keyed by host address, so that only the
// forecast crosses PCIe again.  PCIe, not HBM, bounds these paths.
//
// Cache contract: a cached slab is identified by (host address, byte length);
// the caller promises not to modify cached host arrays while the cache is
// enabled (wb2_set_slab_cache(ctx, 0) drops everything).  Off by default.
#include <algorithm>
#include <unordered_map>

#include "stage.cuh"

namespace wb2 {

int det_metrics_impl(wb2_ctx* ctx, int mode, const void* f, const void* t, const void* c,
                     const void* g, int dtype, int64_t nfield, const int64_t* off_f,
                     const int64_t* off_t, const int64_t* off_c, const int64_t* off_g,
                     const wb2_weights* w, int skipna, double* out);
int spectrum_latsum_impl(wb2_ctx* ctx, const float* x, int64_t nfield, int32_t nrow,
                         int32_t ncol, const double* scale, float* out, int64_t nfield_out,
                         int accumulate);

// Staged slabs and results start 64 elements apart, which keeps them 256-B
// aligned for the kernels.
static int64_t pad64(int64_t elems) { return (elems + 63) / 64 * 64; }

// A 2-D slab of a metric entry's weight grid: `copy` bytes cross PCIe, and
// slabs lie `bytes` (`pad` elements) apart in staging and in the slab cache.
struct SlabGeom {
  int64_t pad;
  size_t bytes, copy;
  SlabGeom(const wb2_weights* w, size_t esize) {
    const int64_t elems = int64_t(w->nrow - 1) * w->row_stride + w->ncol;
    pad = pad64(elems);
    bytes = size_t(pad) * esize;
    copy = size_t(elems) * esize;
  }
};

// Grows the context's staging pair to WB2_STAGE_MB (256 by default), or to
// `min_units` units of `unit` bytes when that is more; the pair is kept for
// later calls.  *units = how many units one buffer holds (at least min_units).
static int stage_units(wb2_ctx* ctx, size_t unit, int64_t* units, int64_t min_units = 1) {
  const char* env = getenv("WB2_STAGE_MB");
  size_t mb = env ? strtoull(env, nullptr, 10) : 256;
  if (mb < 1) mb = 1;
  const size_t need = std::max(mb << 20, unit * size_t(min_units));
  if (ctx->stage_cap < need) {
    WB2_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    WB2_CUDA_TRY(cudaStreamSynchronize(ctx->copy_stream));
    for (void*& b : ctx->stage) {
      if (b) WB2_CUDA_TRY(cudaFree(b));
      b = nullptr;
    }
    ctx->stage_cap = 0;
    for (void*& b : ctx->stage) WB2_CUDA_TRY(cudaMalloc(&b, need));
    ctx->stage_cap = need;
  }
  *units = int64_t(ctx->stage_cap / unit);
  return WB2_OK;
}

// Runs `groups(pipe)` over the context's staging pair with ctx->d_out_tmp
// grown to `bytes`: the whole result, which the groups write part by part on
// the device and which goes back to `out_host` in one copy after the last one.
template <typename Groups>
static int stream_into_result(wb2_ctx* ctx, void* out_host, size_t bytes, Groups&& groups) {
  WB2_TRY(grow_buffer(ctx, ctx->d_out_tmp, ctx->out_tmp_cap, bytes));
  StagePipe pipe(ctx, ctx->stage[0], ctx->stage[1]);
  WB2_TRY(groups(pipe));
  WB2_TRY(pipe.d2h(out_host, ctx->d_out_tmp, bytes));
  return pipe.finish();
}

// Streams `nfield` whole fields through the context's staging pair, as many
// per group as fit at `field_bytes` each: `group(pipe, stage, g0, n)` copies
// fields g0 .. g0 + n - 1 into `stage`, calls pipe.ready(), launches, and
// copies the group's results out.
template <typename Group>
static int stream_field_groups(wb2_ctx* ctx, int64_t nfield, size_t field_bytes, Group&& group) {
  int64_t fpg;
  WB2_TRY(stage_units(ctx, field_bytes, &fpg));
  StagePipe pipe(ctx, ctx->stage[0], ctx->stage[1]);
  for (int64_t g0 = 0; g0 < nfield; g0 += fpg) {
    float* stage;
    WB2_TRY(pipe.next(&stage));
    WB2_TRY(group(pipe, stage, g0, std::min(fpg, nfield - g0)));
    WB2_TRY(pipe.done());
  }
  return pipe.finish();
}

struct SlabCache {
  char* arena = nullptr;
  size_t arena_bytes = 0;
  size_t slab_bytes = 0;  // slot size the arena is currently carved into
  int64_t nslots = 0;
  std::unordered_map<const void*, int64_t> slot_of;
  std::vector<const void*> owner;
  std::vector<uint64_t> last_use;  // group tick of the last kernel that read the slot
  uint64_t tick = 1;
};

void slab_cache_destroy(wb2_ctx* ctx) {
  SlabCache* c = static_cast<SlabCache*>(ctx->slab_cache);
  if (!c) return;
  if (c->arena) cudaFree(c->arena);
  delete c;
  ctx->slab_cache = nullptr;
}

// (Re)carves the arena for slabs of `slab_bytes`; *out = nullptr when the
// cache is disabled or too small for even a few slabs.
static int cache_for(wb2_ctx* ctx, size_t slab_bytes, SlabCache** out) {
  *out = nullptr;
  if (ctx->slab_cache_capacity < 4 * slab_bytes) return WB2_OK;
  SlabCache* c = static_cast<SlabCache*>(ctx->slab_cache);
  if (!c) {
    c = new SlabCache();
    ctx->slab_cache = c;
  }
  if (!c->arena) {
    cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&c->arena), ctx->slab_cache_capacity);
    if (e != cudaSuccess) {
      set_error("slab cache: cudaMalloc(%zu) failed: %s", ctx->slab_cache_capacity,
                cudaGetErrorString(e));
      (void)cudaGetLastError();
      return WB2_ENOMEM;
    }
    c->arena_bytes = ctx->slab_cache_capacity;
    c->slab_bytes = 0;
  }
  if (c->slab_bytes != slab_bytes) {  // another grid: start over
    c->slab_bytes = slab_bytes;
    c->nslots = static_cast<int64_t>(c->arena_bytes / slab_bytes);
    c->slot_of.clear();
    c->owner.assign(c->nslots, nullptr);
    c->last_use.assign(c->nslots, 0);
  }
  *out = c;
  return WB2_OK;
}

// The slab-cache placement of one group of a metric entry.  The group reads
// its slots under one tick.  Its H2D copies (cache fills, and the staged slabs
// the entry queues) go out in placement order, and only once the group knows
// whether a fill refills a slot that the previous group -- the kernels of the
// other staging buffer -- still reads.
struct SlabPlacement {
  struct Copy { const char* src; char* dst; };
  wb2_ctx* ctx;
  SlabCache* cache;  // nullptr: cache off
  const SlabGeom& geom;
  uint64_t tick;
  bool wait_prev = false;
  std::vector<Copy> copies;

  SlabPlacement(wb2_ctx* ctx, SlabCache* cache, const SlabGeom& geom)
      : ctx(ctx), cache(cache), geom(geom), tick(cache ? cache->tick++ : 0) {}
  bool cached(const char* src) const { return cache && cache->slot_of.count(src); }
  void queue(const char* src, char* dst) { copies.push_back({src, dst}); }

  // The slot that holds `src` for this group, or nullptr when the cache is off
  // or every slot is read by this group.  A miss takes a free slot, else the
  // least recently used one, and queues its fill.
  char* place(const char* src) {
    if (!cache) return nullptr;
    SlabCache& c = *cache;
    auto it = c.slot_of.find(src);
    if (it != c.slot_of.end()) {
      c.last_use[it->second] = tick;
      ctx->stat_cache_hits += 1;
      return c.arena + size_t(it->second) * geom.bytes;
    }
    int64_t best = -1;
    uint64_t best_tick = ~uint64_t(0);
    for (int64_t s = 0; s < c.nslots; ++s) {
      if (c.owner[s] == nullptr) {
        best = s;
        best_tick = 0;
        break;
      }
      if (c.last_use[s] < best_tick) {
        best_tick = c.last_use[s];
        best = s;
      }
    }
    if (best < 0 || best_tick >= tick) return nullptr;
    if (c.owner[best]) c.slot_of.erase(c.owner[best]);
    c.owner[best] = src;
    c.slot_of[src] = best;
    const uint64_t prev = c.last_use[best];  // 0: never read
    if (prev + 1 >= tick && prev != 0) wait_prev = true;  // the previous group read it
    c.last_use[best] = tick;
    ctx->stat_cache_misses += 1;
    char* dev = c.arena + size_t(best) * geom.bytes;
    queue(src, dev);
    return dev;
  }
  int issue(StagePipe& pipe) {
    if (wait_prev) WB2_TRY(pipe.wait_other());
    for (const Copy& cp : copies) WB2_TRY(pipe.h2d(cp.dst, cp.src, geom.copy));
    return WB2_OK;
  }
};

}  // namespace wb2

using namespace wb2;

extern "C" {

int wb2_set_slab_cache(wb2_ctx* ctx, size_t bytes) {
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  DeviceGuard g(ctx->device);
  WB2_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  WB2_CUDA_TRY(cudaStreamSynchronize(ctx->copy_stream));
  slab_cache_destroy(ctx);
  ctx->slab_cache_capacity = bytes;
  return WB2_OK;
}

int64_t wb2_transfer_stats(const wb2_ctx* ctx, int which) {
  if (!ctx) return 0;
  switch (which) {
    case 0: return ctx->stat_h2d_bytes;
    case 1: return ctx->stat_d2h_bytes;
    case 2: return ctx->stat_cache_hits;
    case 3: return ctx->stat_cache_misses;
    default: return 0;
  }
}

int wb2_reset_transfer_stats(wb2_ctx* ctx) {
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  ctx->stat_h2d_bytes = ctx->stat_d2h_bytes = 0;
  ctx->stat_cache_hits = ctx->stat_cache_misses = 0;
  return WB2_OK;
}

// ---- K1 -----------------------------------------------------------------------
int wb2_det_metrics_host(wb2_ctx* ctx, const void* f, const void* t, const void* c, int dtype,
                         int64_t nfield, const int64_t* off_f, const int64_t* off_t,
                         const int64_t* off_c, const wb2_weights* w, int skipna,
                         double* out_host) {
  WB2_NVTX("wb2_det_metrics_host");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_REQUIRE(dtype == WB2_F32 || dtype == WB2_F64, "dtype must be WB2_F32 or WB2_F64");
  WB2_TRY(validate_weights(w));
  WB2_REQUIRE(out_host != nullptr, "out is NULL");
  if (nfield == 0) return WB2_OK;
  WB2_REQUIRE(f && t && off_f && off_t, "f/t and their offset tables must not be NULL");
  if (c) WB2_REQUIRE(off_c != nullptr, "climatology offsets are NULL");
  DeviceGuard guard(ctx->device);

  const size_t esize = dtype == WB2_F32 ? 4 : 8;
  const int noper = c ? 3 : 2;
  const SlabGeom geom(w, esize);
  int64_t max_slabs;
  // (an eviction can turn an expected cache hit of the same field into a staged
  // slab: keep `noper` slots of slack)
  WB2_TRY(stage_units(ctx, geom.bytes, &max_slabs, 2 * noper));
  const size_t per_field = size_t(w->nregion) * WB2_DET_NSTAT;
  // the forecast (operand 0) changes every chunk; truth and climatology slabs repeat
  const char* base[3] = {static_cast<const char*>(f), static_cast<const char*>(t),
                         static_cast<const char*>(c)};
  const int64_t* off[3] = {off_f, off_t, off_c};
  return stream_into_result(ctx, out_host, size_t(nfield) * per_field * sizeof(double),
                            [&](StagePipe& pipe) -> int {
    SlabCache* cache;
    WB2_TRY(cache_for(ctx, geom.bytes, &cache));
    std::vector<int64_t> loc[3];
    for (int64_t g0 = 0, g1; g0 < nfield; g0 = g1) {
      char* stage;
      WB2_TRY(pipe.next(&stage));
      SlabPlacement slabs(ctx, cache, geom);
      std::unordered_map<const char*, int64_t> slot_of;  // staged host address -> staging slot
      for (int o = 0; o < noper; ++o) loc[o].clear();
      for (g1 = g0; g1 < nfield; ++g1) {
        // slabs of this field that would have to go through the staging buffer
        const char* src[3];
        int fresh = 0;
        for (int o = 0; o < noper; ++o) {
          src[o] = base[o] + off[o][g1] * esize;
          if (!(o > 0 && slabs.cached(src[o])) && !slot_of.count(src[o])) ++fresh;
        }
        // (a cacheable miss may still land in the cache; counting it against
        // the staging buffer keeps the group bounded either way)
        if (int64_t(slot_of.size()) + fresh > max_slabs - noper) break;
        for (int o = 0; o < noper; ++o) {
          char* dev = o > 0 ? slabs.place(src[o]) : nullptr;
          if (!dev) {
            auto it = slot_of.find(src[o]);
            if (it == slot_of.end()) {
              it = slot_of.emplace(src[o], int64_t(slot_of.size())).first;
              slabs.queue(src[o], stage + size_t(it->second) * geom.bytes);
            }
            dev = stage + size_t(it->second) * geom.bytes;
          }
          loc[o].push_back((dev - stage) / static_cast<int64_t>(esize));
        }
      }
      WB2_REQUIRE(g1 > g0, "staging buffer too small for one field");
      WB2_TRY(slabs.issue(pipe));
      WB2_TRY(pipe.ready());
      WB2_TRY(det_metrics_impl(ctx, c ? 1 : 0, stage, stage, c ? stage : nullptr, nullptr,
                               dtype, g1 - g0, loc[0].data(), loc[1].data(),
                               c ? loc[2].data() : nullptr, nullptr, w, skipna,
                               ctx->d_out_tmp + size_t(g0) * per_field));
      WB2_TRY(pipe.done());
    }
    return WB2_OK;
  });
}

// ---- K2 -----------------------------------------------------------------------
int wb2_ens_metrics_host(wb2_ctx* ctx, const void* x, const void* t, int dtype,
                         int32_t nmember, int64_t member_stride, int64_t nfield,
                         const int64_t* off_x, const int64_t* off_t, const wb2_weights* w,
                         int skipna, double* out_host) {
  WB2_NVTX("wb2_ens_metrics_host");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_REQUIRE(dtype == WB2_F32, "wb2_ens_metrics_host: only WB2_F32 inputs are supported");
  WB2_REQUIRE(nmember >= 1, "wb2_ens_metrics_host: nmember must be >= 1");
  WB2_TRY(validate_weights(w));
  WB2_REQUIRE(out_host != nullptr, "out is NULL");
  if (nfield == 0) return WB2_OK;
  WB2_REQUIRE(x && t && off_x && off_t, "x/t and their offset tables must not be NULL");
  DeviceGuard guard(ctx->device);

  const size_t esize = 4;
  const SlabGeom geom(w, esize);
  const int64_t per = int64_t(nmember) + 1;  // staging slots per field (members + truth)
  int64_t fields_per_group;
  WB2_TRY(stage_units(ctx, geom.bytes * size_t(per), &fields_per_group));
  const size_t per_field = size_t(w->nregion) * WB2_ENS_NSTAT;
  const char* xh = static_cast<const char*>(x);
  const char* th = static_cast<const char*>(t);
  return stream_into_result(ctx, out_host, size_t(nfield) * per_field * sizeof(double),
                            [&](StagePipe& pipe) -> int {
    SlabCache* cache;
    WB2_TRY(cache_for(ctx, geom.bytes, &cache));
    std::vector<int64_t> lx, lt;
    for (int64_t g0 = 0; g0 < nfield; g0 += fields_per_group) {
      const int64_t g1 = std::min(nfield, g0 + fields_per_group);
      char* stage;
      WB2_TRY(pipe.next(&stage));
      SlabPlacement truth(ctx, cache, geom);
      lx.clear();
      lt.clear();
      for (int64_t i = g0; i < g1; ++i) {
        char* fbase = stage + size_t(i - g0) * size_t(per) * geom.bytes;
        // the members go out at once: they land in this group's staging
        // buffer, which pipe.next() has ordered after the kernels that read it
        for (int m = 0; m < nmember; ++m)
          WB2_TRY(pipe.h2d(fbase + size_t(m) * geom.bytes,
                           xh + (off_x[i] + int64_t(m) * member_stride) * int64_t(esize),
                           geom.copy));
        lx.push_back((fbase - stage) / int64_t(esize));
        const char* tsrc = th + off_t[i] * int64_t(esize);
        char* tdev = truth.place(tsrc);
        if (!tdev) truth.queue(tsrc, tdev = fbase + size_t(nmember) * geom.bytes);
        lt.push_back((tdev - stage) / int64_t(esize));
      }
      WB2_TRY(truth.issue(pipe));
      WB2_TRY(pipe.ready());
      WB2_TRY(wb2_ens_metrics(ctx, stage, stage, WB2_F32, nmember, geom.pad, g1 - g0,
                              lx.data(), lt.data(), w, skipna,
                              ctx->d_out_tmp + size_t(g0) * per_field));
      WB2_TRY(pipe.done());
    }
    return WB2_OK;
  });
}

// ---- K5 -----------------------------------------------------------------------
int wb2_regrid_conservative_host(wb2_ctx* ctx, const float* src, float* dst, int64_t nfield,
                                 int64_t src_field_stride, int64_t dst_field_stride,
                                 const wb2_csr* lon_w, const wb2_csr* lat_w) {
  WB2_NVTX("wb2_regrid_conservative_host");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_REQUIRE(lon_w && lat_w, "weights are NULL");
  WB2_REQUIRE(nfield >= 0, "nfield < 0");
  if (nfield == 0) return WB2_OK;
  WB2_REQUIRE(src && dst, "src/dst are NULL");
  const int64_t in_elems = int64_t(lon_w->n_src) * lat_w->n_src;
  const int64_t out_elems = int64_t(lon_w->n_tgt) * lat_w->n_tgt;
  WB2_REQUIRE(src_field_stride >= in_elems && dst_field_stride >= out_elems,
              "field strides smaller than a slab");
  DeviceGuard guard(ctx->device);
  const int64_t in_pad = pad64(in_elems), out_pad = pad64(out_elems);
  return stream_field_groups(ctx, nfield, size_t(in_pad + out_pad) * 4,
                             [&](StagePipe& pipe, float* sin, int64_t g0, int64_t n) -> int {
    float* sout = sin + size_t(n) * in_pad;
    // one 2-D copy for the whole group (pitch = the caller's field stride)
    WB2_TRY(pipe.h2d_2d(sin, size_t(in_pad) * 4, src + g0 * src_field_stride,
                        size_t(src_field_stride) * 4, size_t(in_elems) * 4, size_t(n)));
    WB2_TRY(pipe.ready());
    WB2_TRY(wb2_regrid_conservative(ctx, sin, sout, n, in_pad, out_pad, lon_w, lat_w));
    return pipe.d2h_2d(dst + g0 * dst_field_stride, size_t(dst_field_stride) * 4, sout,
                       size_t(out_pad) * 4, size_t(out_elems) * 4, size_t(n));
  });
}

// ---- K4 -----------------------------------------------------------------------
// reduce: 0 = per-latitude spectra (wb2_zonal_spectrum), 1 = latitude-weighted
// reduction (wb2_zonal_spectrum_latsum; accumulate is implied).
static int spectrum_host(wb2_ctx* ctx, const float* x, int64_t nfield, int32_t nrow,
                         int32_t ncol, const double* scale, float* out_host,
                         int32_t accumulate, int64_t nfield_out, int reduce) {
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_REQUIRE(nrow > 0 && ncol > 1, "bad grid %d x %d", nrow, ncol);
  WB2_REQUIRE(nfield >= 0, "nfield < 0");
  if (nfield == 0) return WB2_OK;
  WB2_REQUIRE(x && out_host && scale, "NULL argument");
  if (!accumulate && !reduce) nfield_out = nfield;
  WB2_REQUIRE(nfield_out > 0 && nfield % nfield_out == 0,
              "nfield (%lld) must be a multiple of nfield_out (%lld)",
              static_cast<long long>(nfield), static_cast<long long>(nfield_out));
  DeviceGuard guard(ctx->device);
  const int nk = ncol / 2 + 1;
  const int64_t in_elems = int64_t(nrow) * ncol;  // multiple of 4 floats whenever ncol is even
  const int64_t out_elems = reduce ? nk : int64_t(nrow) * nk;
  const int64_t ntimes = nfield / nfield_out;

  if (!accumulate && !reduce) {
    // fields in, spectra out, group by group
    return stream_field_groups(ctx, nfield, size_t(pad64(in_elems) + pad64(out_elems)) * 4,
                               [&](StagePipe& pipe, float* sin, int64_t g0, int64_t n) -> int {
      // rows stay contiguous: in_elems per field, no padding between fields
      WB2_TRY(pipe.h2d(sin, x + g0 * in_elems, size_t(n) * in_elems * 4));
      WB2_TRY(pipe.ready());
      float* sout = sin + pad64(n * in_elems);
      WB2_TRY(wb2_zonal_spectrum(ctx, sin, n, nrow, ncol, scale, sout, 0, n));
      return pipe.d2h(out_host + g0 * out_elems, sout, size_t(n) * out_elems * 4);
    });
  }

  // time-summed / latitude-reduced: the accumulator stays on the device.  A
  // group = `k` time steps of a run of `S` slots (slot-minor, like the device
  // entry), so every launch adds whole time steps to its slots.
  int64_t fit;
  WB2_TRY(stage_units(ctx, size_t(in_elems) * 4, &fit));
  const int64_t S = std::min(nfield_out, fit);
  const int64_t k = fit / S;
  const size_t acc_bytes = size_t(nfield_out) * out_elems * 4;
  // the device accumulator lives in out_tmp (scratch is used by the kernels)
  return stream_into_result(ctx, out_host, acc_bytes, [&](StagePipe& pipe) -> int {
    float* acc = reinterpret_cast<float*>(ctx->d_out_tmp);
    WB2_CUDA_TRY(cudaMemsetAsync(acc, 0, acc_bytes, ctx->stream));
    for (int64_t s0 = 0; s0 < nfield_out; s0 += S) {
      const int64_t ns = std::min(S, nfield_out - s0);
      for (int64_t t0 = 0; t0 < ntimes; t0 += k) {
        const int64_t nt = std::min(k, ntimes - t0);
        float* sin;
        WB2_TRY(pipe.next(&sin));
        // per time step a contiguous run of ns fields
        for (int64_t ti = 0; ti < nt; ++ti)
          WB2_TRY(pipe.h2d(sin + ti * ns * in_elems,
                           x + ((t0 + ti) * nfield_out + s0) * in_elems,
                           size_t(ns) * in_elems * 4));
        WB2_TRY(pipe.ready());
        if (reduce)
          WB2_TRY(spectrum_latsum_impl(ctx, sin, nt * ns, nrow, ncol, scale,
                                       acc + s0 * out_elems, ns, 1));
        else
          WB2_TRY(wb2_zonal_spectrum(ctx, sin, nt * ns, nrow, ncol, scale,
                                     acc + s0 * out_elems, 1, ns));
        WB2_TRY(pipe.done());
      }
    }
    return WB2_OK;
  });
}

int wb2_zonal_spectrum_host(wb2_ctx* ctx, const float* x, int64_t nfield, int32_t nrow,
                            int32_t ncol, const double* scale, float* out_host,
                            int32_t accumulate, int64_t nfield_out) {
  WB2_NVTX("wb2_zonal_spectrum_host");
  return spectrum_host(ctx, x, nfield, nrow, ncol, scale, out_host, accumulate, nfield_out, 0);
}

int wb2_zonal_spectrum_latsum_host(wb2_ctx* ctx, const float* x, int64_t nfield, int32_t nrow,
                                   int32_t ncol, const double* scale, float* out_host,
                                   int64_t nfield_out) {
  WB2_NVTX("wb2_zonal_spectrum_latsum_host");
  return spectrum_host(ctx, x, nfield, nrow, ncol, scale, out_host, 1, nfield_out, 1);
}

}  // extern "C"

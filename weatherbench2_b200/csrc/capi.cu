// Context management and memory helpers of the C ABI (include/wb2b200.h).
#include "common.cuh"

namespace wb2 {

static thread_local char g_err[1024] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int Packer::commit() {
  Slot& s = ctx_->slots[ctx_->next_slot];
  ctx_->next_slot = (ctx_->next_slot + 1) % kNumSlots;
  if (s.used) {
    // wait until the kernels that read this slot's device block are done
    WB2_CUDA_TRY(cudaEventSynchronize(s.done));
  }
  size_t upload_end = 0;
  for (const Item& it : items_)
    if (it.src) upload_end = it.off + it.bytes;
  size_t need = (size_ + 255) & ~size_t(255);
  if (need > s.dcap) {
    size_t cap = need + need / 2 + 4096;
    if (s.d) WB2_CUDA_TRY(cudaFree(s.d));
    s.d = nullptr;
    s.dcap = 0;
    WB2_CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(&s.d), cap));
    s.dcap = cap;
  }
  if (upload_end > s.hcap) {
    size_t cap = upload_end + upload_end / 2 + 4096;
    if (s.h) WB2_CUDA_TRY(cudaFreeHost(s.h));
    s.h = nullptr;
    s.hcap = 0;
    WB2_CUDA_TRY(cudaMallocHost(reinterpret_cast<void**>(&s.h), cap));
    s.hcap = cap;
  }
  if (!s.done) WB2_CUDA_TRY(cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming));
  // Upload only the prefix that holds host data (scratch reservations that
  // follow the last uploaded item are not copied).
  for (const Item& it : items_)
    if (it.src) memcpy(s.h + it.off, it.src, it.bytes);
  if (upload_end) {
    WB2_CUDA_TRY(cudaMemcpyAsync(s.d, s.h, upload_end, cudaMemcpyHostToDevice,
                                 ctx_->stream));
  }
  s.used = true;
  slot_ = &s;
  return WB2_OK;
}

int Packer::release() {
  if (slot_) WB2_CUDA_TRY(cudaEventRecord(slot_->done, ctx_->stream));
  return WB2_OK;
}

int validate_weights(const wb2_weights* w) {
  WB2_REQUIRE(w != nullptr, "weights descriptor is NULL");
  WB2_REQUIRE(w->nrow > 0 && w->ncol > 0, "weights: nrow/ncol must be > 0");
  WB2_REQUIRE(w->row_stride >= w->ncol, "weights: row_stride < ncol");
  WB2_REQUIRE(w->nregion >= 1 && w->nregion <= WB2_MAX_REGIONS,
              "weights: nregion must be in 1..%d (got %d)", WB2_MAX_REGIONS,
              w->nregion);
  WB2_REQUIRE(w->nseg >= 1 && w->nseg <= w->ncol, "weights: bad nseg %d", w->nseg);
  WB2_REQUIRE(w->row_w && w->seg_start && w->seg_w,
              "weights: row_w / seg_start / seg_w must not be NULL");
  WB2_REQUIRE(w->seg_start[0] == 0 && w->seg_start[w->nseg] == w->ncol,
              "weights: seg_start must cover [0, ncol)");
  for (int k = 0; k < w->nseg; ++k)
    WB2_REQUIRE(w->seg_start[k] < w->seg_start[k + 1],
                "weights: seg_start must be strictly increasing");
  // The kernels skip cells whose weight == 0, the reference those whose
  // weight is not > 0: the two agree only without negative weights.  (cell_w
  // is a device array and is not checked here.)
  if (w->zero_skip) {
    for (int64_t i = 0; i < int64_t(w->nregion) * w->nrow; ++i)
      WB2_REQUIRE(!(w->row_w[i] < 0), "weights: zero_skip needs non-negative weights "
                  "(row_w[%lld] = %g)", static_cast<long long>(i), w->row_w[i]);
    for (int64_t i = 0; i < int64_t(w->nregion) * w->nseg; ++i)
      WB2_REQUIRE(!(w->seg_w[i] < 0), "weights: zero_skip needs non-negative weights "
                  "(seg_w[%lld] = %g)", static_cast<long long>(i), w->seg_w[i]);
    for (int i = 0; w->col_w && i < w->ncol; ++i)
      WB2_REQUIRE(!(w->col_w[i] < 0), "weights: zero_skip needs non-negative weights "
                  "(col_w[%d] = %g)", i, static_cast<double>(w->col_w[i]));
  }
  return WB2_OK;
}

}  // namespace wb2

using namespace wb2;

extern "C" {

int wb2_version(void) { return WB2_VERSION; }
const char* wb2_last_error(void) { return g_err; }
int wb2_has_cuda(void) { return 1; }
int64_t wb2_launch_count(const wb2_ctx* ctx) { return ctx ? ctx->launches : 0; }

int wb2_create(int device, wb2_ctx** out) {
  WB2_REQUIRE(out != nullptr, "wb2_create: out is NULL");
  *out = nullptr;
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    set_error("wb2_create: no CUDA device available (%s)",
              e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    return WB2_ECUDA;
  }
  WB2_REQUIRE(device >= 0 && device < ndev, "wb2_create: bad device %d (have %d)",
              device, ndev);
  DeviceGuard g(device);
  cudaDeviceProp prop;
  WB2_CUDA_TRY(cudaGetDeviceProperties(&prop, device));
  // sm_90a code runs on compute capability 9.0 only (arch-specific features:
  // no forward compatibility to later architectures)
  if (prop.major != 9 || prop.minor != 0) {
    set_error("wb2_create: device %d is sm_%d%d; this library is built for sm_90a only",
              device, prop.major, prop.minor);
    return WB2_EUNSUPPORTED;
  }
  wb2_ctx* c = new wb2_ctx();
  c->device = device;
  c->num_sms = prop.multiProcessorCount;
  WB2_CUDA_TRY(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
  WB2_CUDA_TRY(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
  for (int i = 0; i < 2; ++i) {
    WB2_CUDA_TRY(cudaEventCreateWithFlags(&c->stage_copied[i], cudaEventDisableTiming));
    WB2_CUDA_TRY(cudaEventCreateWithFlags(&c->stage_free[i], cudaEventDisableTiming));
  }
  *out = c;
  return WB2_OK;
}

int wb2_destroy(wb2_ctx* c) {
  if (!c) return WB2_OK;
  DeviceGuard g(c->device);
  cudaStreamSynchronize(c->stream);
  cudaStreamSynchronize(c->copy_stream);
  for (auto& s : c->slots) {
    if (s.h) cudaFreeHost(s.h);
    if (s.d) cudaFree(s.d);
    if (s.done) cudaEventDestroy(s.done);
  }
  for (int i = 0; i < 2; ++i) {
    if (c->stage[i]) cudaFree(c->stage[i]);
    if (c->stage_copied[i]) cudaEventDestroy(c->stage_copied[i]);
    if (c->stage_free[i]) cudaEventDestroy(c->stage_free[i]);
  }
  slab_cache_destroy(c);
  if (c->order_in) cudaEventDestroy(c->order_in);
  if (c->order_out) cudaEventDestroy(c->order_out);
  if (c->d_out_tmp) cudaFree(c->d_out_tmp);
  if (c->tma_partial) cudaFree(c->tma_partial);
  if (c->scratch) cudaFree(c->scratch);
  if (c->own_stream && c->stream) cudaStreamDestroy(c->stream);
  if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
  delete c;
  return WB2_OK;
}

int wb2_set_stream(wb2_ctx* c, void* cuda_stream) {
  WB2_REQUIRE(c != nullptr, "ctx is NULL");
  DeviceGuard g(c->device);
  WB2_CUDA_TRY(cudaStreamSynchronize(c->stream));
  if (c->own_stream && c->stream) cudaStreamDestroy(c->stream);
  if (cuda_stream) {
    c->stream = reinterpret_cast<cudaStream_t>(cuda_stream);
    c->own_stream = false;
  } else {
    WB2_CUDA_TRY(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    c->own_stream = true;
  }
  return WB2_OK;
}

void* wb2_get_stream(wb2_ctx* c) { return c ? reinterpret_cast<void*>(c->stream) : nullptr; }

int wb2_synchronize(wb2_ctx* c) {
  WB2_REQUIRE(c != nullptr, "ctx is NULL");
  DeviceGuard g(c->device);
  WB2_CUDA_TRY(cudaStreamSynchronize(c->stream));
  return WB2_OK;
}

int wb2_wait_stream(wb2_ctx* c, void* cuda_stream) {
  WB2_REQUIRE(c != nullptr, "ctx is NULL");
  cudaStream_t other = reinterpret_cast<cudaStream_t>(cuda_stream);
  if (other == c->stream) return WB2_OK;  // same stream: already ordered
  DeviceGuard g(c->device);
  if (!c->order_in)
    WB2_CUDA_TRY(cudaEventCreateWithFlags(&c->order_in, cudaEventDisableTiming));
  WB2_CUDA_TRY(cudaEventRecord(c->order_in, other));
  WB2_CUDA_TRY(cudaStreamWaitEvent(c->stream, c->order_in, 0));
  WB2_CUDA_TRY(cudaStreamWaitEvent(c->copy_stream, c->order_in, 0));
  return WB2_OK;
}

int wb2_stream_wait(wb2_ctx* c, void* cuda_stream) {
  WB2_REQUIRE(c != nullptr, "ctx is NULL");
  cudaStream_t other = reinterpret_cast<cudaStream_t>(cuda_stream);
  if (other == c->stream) return WB2_OK;
  DeviceGuard g(c->device);
  if (!c->order_out)
    WB2_CUDA_TRY(cudaEventCreateWithFlags(&c->order_out, cudaEventDisableTiming));
  WB2_CUDA_TRY(cudaEventRecord(c->order_out, c->stream));
  WB2_CUDA_TRY(cudaStreamWaitEvent(other, c->order_out, 0));
  return WB2_OK;
}

int wb2_malloc(wb2_ctx* c, size_t bytes, void** p) {
  WB2_REQUIRE(c && p, "wb2_malloc: NULL argument");
  DeviceGuard g(c->device);
  WB2_CUDA_TRY(cudaMalloc(p, bytes ? bytes : 1));
  return WB2_OK;
}
int wb2_free(wb2_ctx* c, void* p) {
  WB2_REQUIRE(c != nullptr, "ctx is NULL");
  DeviceGuard g(c->device);
  WB2_CUDA_TRY(cudaStreamSynchronize(c->stream));
  WB2_CUDA_TRY(cudaFree(p));
  return WB2_OK;
}
int wb2_host_alloc(wb2_ctx* c, size_t bytes, void** p) {
  WB2_REQUIRE(c && p, "wb2_host_alloc: NULL argument");
  DeviceGuard g(c->device);
  WB2_CUDA_TRY(cudaMallocHost(p, bytes ? bytes : 1));
  return WB2_OK;
}
int wb2_host_free(wb2_ctx* c, void* p) {
  WB2_REQUIRE(c != nullptr, "ctx is NULL");
  DeviceGuard g(c->device);
  WB2_CUDA_TRY(cudaFreeHost(p));
  return WB2_OK;
}
int wb2_memcpy_h2d(wb2_ctx* c, void* d, const void* h, size_t bytes) {
  WB2_REQUIRE(c != nullptr, "ctx is NULL");
  DeviceGuard g(c->device);
  WB2_CUDA_TRY(cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, c->stream));
  WB2_CUDA_TRY(cudaStreamSynchronize(c->stream));
  return WB2_OK;
}
int wb2_memcpy_d2h(wb2_ctx* c, void* h, const void* d, size_t bytes) {
  WB2_REQUIRE(c != nullptr, "ctx is NULL");
  DeviceGuard g(c->device);
  WB2_CUDA_TRY(cudaMemcpyAsync(h, d, bytes, cudaMemcpyDeviceToHost, c->stream));
  WB2_CUDA_TRY(cudaStreamSynchronize(c->stream));
  return WB2_OK;
}
int wb2_memset(wb2_ctx* c, void* d, int value, size_t bytes) {
  WB2_REQUIRE(c != nullptr, "ctx is NULL");
  DeviceGuard g(c->device);
  WB2_CUDA_TRY(cudaMemsetAsync(d, value, bytes, c->stream));
  return WB2_OK;
}

}  // extern "C"

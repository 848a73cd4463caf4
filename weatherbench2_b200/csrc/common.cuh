// Shared internals of libwb2b200.so (sm_90a).  Not part of the C ABI.
#pragma once

#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>

#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/wb2b200.h"

namespace wb2 {

void set_error(const char* fmt, ...);

#define WB2_CUDA_TRY(expr)                                                    \
  do {                                                                        \
    cudaError_t _e = (expr);                                                  \
    if (_e != cudaSuccess) {                                                  \
      ::wb2::set_error("%s failed at %s:%d: %s", #expr, __FILE__, __LINE__,   \
                       cudaGetErrorString(_e));                               \
      return WB2_ECUDA;                                                       \
    }                                                                         \
  } while (0)

#define WB2_REQUIRE(cond, ...)                                                \
  do {                                                                        \
    if (!(cond)) {                                                            \
      ::wb2::set_error(__VA_ARGS__);                                          \
      return WB2_EINVAL;                                                      \
    }                                                                         \
  } while (0)

#define WB2_TRY(expr)                                                         \
  do {                                                                        \
    int _rc = (expr);                                                         \
    if (_rc != WB2_OK) return _rc;                                            \
  } while (0)

// One descriptor-upload slot: a pinned host staging block, its device twin and
// an event that marks "the last kernel that read the device block finished".
struct Slot {
  char* h = nullptr;
  char* d = nullptr;
  size_t hcap = 0;
  size_t dcap = 0;
  cudaEvent_t done = nullptr;
  bool used = false;
};

constexpr int kNumSlots = 4;

}  // namespace wb2

struct wb2_ctx {
  int device = 0;
  int num_sms = 132;
  cudaStream_t stream = nullptr;
  bool own_stream = true;
  cudaStream_t copy_stream = nullptr;
  wb2::Slot slots[wb2::kNumSlots];
  int next_slot = 0;
  int64_t launches = 0;
  // staging for the *_host entry points (double buffered)
  void* stage[2] = {nullptr, nullptr};
  size_t stage_cap = 0;
  cudaEvent_t stage_copied[2] = {nullptr, nullptr};
  cudaEvent_t stage_free[2] = {nullptr, nullptr};
  double* d_out_tmp = nullptr;
  size_t out_tmp_cap = 0;
  // per-(CTA, warp) partials of the TMA-staged K1 kernel
  double* tma_partial = nullptr;
  size_t tma_partial_cap = 0;
  // generic scratch of the other kernels (grown on demand)
  void* scratch = nullptr;
  size_t scratch_cap = 0;
  // cross-stream ordering with a caller's stream (wb2_wait_stream / wb2_stream_wait)
  cudaEvent_t order_in = nullptr;
  cudaEvent_t order_out = nullptr;
  // device-resident LRU cache of host slabs (host_stream.cu); 0 = disabled
  void* slab_cache = nullptr;
  size_t slab_cache_capacity = 0;
  // transfer accounting of the *_host entries (wb2_transfer_stats)
  int64_t stat_h2d_bytes = 0, stat_d2h_bytes = 0;
  int64_t stat_cache_hits = 0, stat_cache_misses = 0;
};

namespace wb2 {

// Packs small host arrays into one slot and uploads them with a single async
// copy.  Usage: Packer p(ctx); off = p.add(ptr, bytes) ...; p.commit(); then
// p.dev(off) gives device pointers;  p.release() records the slot's event after
// the consuming kernels were enqueued.
class Packer {
 public:
  explicit Packer(wb2_ctx* ctx) : ctx_(ctx) {}
  size_t add(const void* src, size_t bytes) {
    size_t off = (size_ + 255) & ~size_t(255);
    items_.push_back({src, off, bytes});
    size_ = off + bytes;
    return off;
  }
  // reserve device-only scratch inside the slot (not uploaded)
  size_t reserve(size_t bytes) { return add(nullptr, bytes); }
  int commit();
  template <typename T>
  T* dev(size_t off) const { return reinterpret_cast<T*>(slot_->d + off); }
  int release();

 private:
  struct Item { const void* src; size_t off; size_t bytes; };
  wb2_ctx* ctx_;
  std::vector<Item> items_;
  size_t size_ = 0;
  Slot* slot_ = nullptr;
};

// NVTX range around every compute entry point of the C ABI (visible in Nsight
// Systems / ncu --nvtx; a no-op when no tool is attached): the trace hook
// SURVEY.md section 5 lists.
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
};
#define WB2_NVTX(name) ::wb2::NvtxRange wb2_nvtx_range_(name)

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    cudaGetDevice(&prev);
    if (prev != dev) cudaSetDevice(dev);
  }
  ~DeviceGuard() {
    int cur = -1;
    cudaGetDevice(&cur);
    if (prev >= 0 && cur != prev) cudaSetDevice(prev);
  }
};

// Grows a device buffer held by the context (`buf`, capacity `cap` bytes) to
// at least `need` bytes; the contents are not kept.  Waits for the kernels
// that may still read the old buffer before freeing it.
template <typename T>
int grow_buffer(wb2_ctx* ctx, T*& buf, size_t& cap, size_t need) {
  if (cap >= need) return WB2_OK;
  WB2_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  if (buf) WB2_CUDA_TRY(cudaFree(buf));
  buf = nullptr;
  cap = 0;
  WB2_CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(&buf), need));
  cap = need;
  return WB2_OK;
}

// Launches `kernel` on the context's stream, first raising its dynamic
// shared-memory limit when `smem` exceeds the default 48 KB.
template <typename... P, typename... A>
int launch_kernel(wb2_ctx* ctx, void (*kernel)(P...), dim3 grid, int block, size_t smem,
                  const A&... args) {
  if (smem > 48 * 1024)
    WB2_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      static_cast<int>(smem)));
  kernel<<<grid, block, smem, ctx->stream>>>(args...);
  WB2_CUDA_TRY(cudaGetLastError());
  return WB2_OK;
}

int validate_weights(const wb2_weights* w);
void slab_cache_destroy(wb2_ctx* ctx);  // host_stream.cu

// ens_big.cu: ensembles of more than 64 members (rank by counting).
int ens_metrics_big(wb2_ctx* ctx, const float* x, const float* t, int32_t nmember,
                    int64_t member_stride, int64_t nfield, const int64_t* off_x,
                    const int64_t* off_t, const wb2_weights* w, int skipna, double* out);

// ---- device helpers ---------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// streaming 128-bit load, bypass L1 allocation (data is touched once)
__device__ __forceinline__ float4 ldg_stream(const float4* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ float ldg_stream(const float* p) {
  float r;
  asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(r) : "l"(p));
  return r;
}
__device__ __forceinline__ double ldg_stream(const double* p) {
  double r;
  asm volatile("ld.global.nc.L1::no_allocate.f64 %0, [%1];" : "=d"(r) : "l"(p));
  return r;
}
__device__ __forceinline__ double2 ldg_stream(const double2* p) {
  double2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.f64 {%0,%1}, [%2];"
               : "=d"(r.x), "=d"(r.y)
               : "l"(p));
  return r;
}

}  // namespace wb2

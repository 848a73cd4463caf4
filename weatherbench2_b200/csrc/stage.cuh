// Host-to-device movement of the C ABI entries: the double-buffered staging
// pipe every *_host entry streams its input through, and one-shot uploads of
// small host tables into device blocks the entry owns.
#pragma once

#include <initializer_list>

#include "common.cuh"

namespace wb2 {

// The ordering protocol of a double-buffered host stream; bands alternate
// between two device buffers that the pipe neither chooses nor owns.  A band:
// next() (the copy stream waits for the kernels that last read the band's
// buffer), h2d* copies on the copy stream, ready() (ctx->stream waits for
// them), the band's kernels and d2h* copies on ctx->stream, done().  So the
// copy of band b+1 overlaps the kernels of band b.  Every copy adds the bytes
// it moves to the context's transfer counters.  finish() waits for ctx->stream
// on the success path; the destructor drains both streams, so no copy is in
// flight once the pipe is gone, whatever path the entry returns by.
class StagePipe {
 public:
  StagePipe(wb2_ctx* ctx, void* buf0, void* buf1)
      : ctx_(ctx), buf_{static_cast<char*>(buf0), static_cast<char*>(buf1)} {}
  StagePipe(const StagePipe&) = delete;
  StagePipe& operator=(const StagePipe&) = delete;
  ~StagePipe() {
    cudaStreamSynchronize(ctx_->stream);
    cudaStreamSynchronize(ctx_->copy_stream);
  }

  template <typename T>
  int next(T** buf) {
    if (used_[cur_])
      WB2_CUDA_TRY(cudaStreamWaitEvent(ctx_->copy_stream, ctx_->stage_free[cur_], 0));
    *buf = reinterpret_cast<T*>(buf_[cur_]);
    return WB2_OK;
  }
  // The copy stream also waits for the kernels of the other buffer (they read
  // a slab-cache slot that this band refills).
  int wait_other() {
    if (used_[cur_ ^ 1])
      WB2_CUDA_TRY(cudaStreamWaitEvent(ctx_->copy_stream, ctx_->stage_free[cur_ ^ 1], 0));
    return WB2_OK;
  }
  int h2d(void* dst, const void* src, size_t bytes) {
    WB2_CUDA_TRY(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx_->copy_stream));
    ctx_->stat_h2d_bytes += int64_t(bytes);
    return WB2_OK;
  }
  int h2d_2d(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width,
             size_t rows) {
    WB2_CUDA_TRY(cudaMemcpy2DAsync(dst, dpitch, src, spitch, width, rows,
                                   cudaMemcpyHostToDevice, ctx_->copy_stream));
    ctx_->stat_h2d_bytes += int64_t(width * rows);
    return WB2_OK;
  }
  int ready() {
    WB2_CUDA_TRY(cudaEventRecord(ctx_->stage_copied[cur_], ctx_->copy_stream));
    WB2_CUDA_TRY(cudaStreamWaitEvent(ctx_->stream, ctx_->stage_copied[cur_], 0));
    return WB2_OK;
  }
  int d2h(void* dst, const void* src, size_t bytes) {
    WB2_CUDA_TRY(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, ctx_->stream));
    ctx_->stat_d2h_bytes += int64_t(bytes);
    return WB2_OK;
  }
  int d2h_2d(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width,
             size_t rows) {
    WB2_CUDA_TRY(cudaMemcpy2DAsync(dst, dpitch, src, spitch, width, rows,
                                   cudaMemcpyDeviceToHost, ctx_->stream));
    ctx_->stat_d2h_bytes += int64_t(width * rows);
    return WB2_OK;
  }
  int done() {
    WB2_CUDA_TRY(cudaEventRecord(ctx_->stage_free[cur_], ctx_->stream));
    used_[cur_] = true;
    cur_ ^= 1;
    return WB2_OK;
  }
  int finish() {
    WB2_CUDA_TRY(cudaStreamSynchronize(ctx_->stream));
    return WB2_OK;
  }

 private:
  wb2_ctx* ctx_;
  char* buf_[2];
  bool used_[2] = {false, false};
  int cur_ = 0;
};

// A staging pair private to one call, for the entries whose bands follow the
// caller's budget: cudaMalloc'd, and cudaFree'd on return.  Declared before
// the pipe that uses it, it is freed after the pipe has drained.
struct StagePair {
  char* buf[2] = {nullptr, nullptr};
  StagePair() = default;
  StagePair(const StagePair&) = delete;
  StagePair& operator=(const StagePair&) = delete;
  ~StagePair() {
    for (char* b : buf)
      if (b) cudaFree(b);
  }
  int alloc(size_t bytes) {
    for (char*& b : buf) WB2_CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(&b), bytes));
    return WB2_OK;
  }
};

// A device block from cudaMallocAsync on ctx->stream, freed with cudaFreeAsync
// on that stream when the owner goes out of scope.
class DeviceBlock {
 public:
  DeviceBlock() = default;
  DeviceBlock(const DeviceBlock&) = delete;
  DeviceBlock& operator=(const DeviceBlock&) = delete;
  ~DeviceBlock() {
    if (p_) cudaFreeAsync(p_, stream_);
  }
  int alloc(wb2_ctx* ctx, size_t bytes) {
    stream_ = ctx->stream;
    WB2_CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&p_), bytes, stream_));
    return WB2_OK;
  }
  template <typename T>
  T* at(size_t off) const { return reinterpret_cast<T*>(p_ + off); }

 private:
  char* p_ = nullptr;
  cudaStream_t stream_ = nullptr;
};

struct HostPart {
  const void* src;  // may be NULL when bytes == 0
  size_t bytes;
};

// Uploads `parts`, each at the next 8-byte-aligned offset (offs[i]), into a
// new block held by `blk`.  They are packed into a pageable vector that goes
// away on return, so the copy is waited for.  (Not a Packer slot: later calls
// of the same entry, such as the wb2_ens_mean calls of the daily resample, can
// recycle those.)
inline int upload_parts(wb2_ctx* ctx, std::initializer_list<HostPart> parts, DeviceBlock* blk,
                        size_t* offs) {
  size_t bytes = 0, i = 0;
  for (const HostPart& part : parts) {
    offs[i++] = bytes = (bytes + 7) / 8 * 8;
    bytes += part.bytes;
  }
  std::vector<char> h(bytes);
  i = 0;
  for (const HostPart& part : parts) {
    if (part.bytes) memcpy(h.data() + offs[i], part.src, part.bytes);
    ++i;
  }
  WB2_TRY(blk->alloc(ctx, bytes));
  WB2_CUDA_TRY(cudaMemcpyAsync(blk->at<char>(0), h.data(), bytes, cudaMemcpyHostToDevice,
                               ctx->stream));
  WB2_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  return WB2_OK;
}

}  // namespace wb2

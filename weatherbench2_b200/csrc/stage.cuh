// Host-to-device movement of the C ABI entries: the double-buffered staging
// pipe every *_host entry streams its input through, and one-shot uploads of
// small host tables into device blocks the entry owns.
#pragma once

#include <algorithm>
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
  // `slices` planes of `rows` rows of `width` bytes into dst, packed; in the
  // source, rows are `spitch` bytes apart and planes `spitch * srows`.
  int h2d_3d(void* dst, const void* src, size_t spitch, size_t srows, size_t width, size_t rows,
             size_t slices) {
    cudaMemcpy3DParms p = {};
    p.srcPtr = make_cudaPitchedPtr(const_cast<void*>(src), spitch, width, srows);
    p.dstPtr = make_cudaPitchedPtr(dst, width, width, rows);
    p.extent = make_cudaExtent(width, rows, slices);
    p.kind = cudaMemcpyHostToDevice;
    WB2_CUDA_TRY(cudaMemcpy3DAsync(&p, ctx_->copy_stream));
    ctx_->stat_h2d_bytes += int64_t(width * rows * slices);
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

// Streams a HOST series [nouter][ntime][ninner] of `es`-byte values through a
// private staging pair in bands: inner cells of one outer index, or whole
// outer indices when one fits `budget` (the device bytes of both buffers, at
// least one cell per band).  Each band is one strided 2-D copy of k outer x n
// inner cells; `launch(in, k, n, dev_out)` runs its kernels on ctx->stream,
// reading `in` as [k][ntime][n] and writing dev_out[s] as [k][nout][n] for
// every s whose out_host[s] is not NULL; those are copied back into
// out_host[s], host [nouter][nout][ninner].  nout_host <= 4.  Outputs are
// `out_es`-byte values.  With `out_major` the band outputs are [nout][k][n]
// instead and the host outputs [nout][nouter][ninner]: a band is part of one
// outer index or whole outer indices, so its cells are one contiguous run of
// every host plane and come back in one 2-D copy.
template <typename Launch>
int stream_series_bands(wb2_ctx* ctx, const void* x, size_t es, size_t out_es, int64_t nouter,
                        int64_t ntime, int64_t ninner, int64_t nout, bool out_major,
                        char* const* out_host, int nout_host, size_t budget, Launch&& launch) {
  int nstat = 0;
  for (int s = 0; s < nout_host; ++s) nstat += out_host[s] != nullptr;
  const size_t per_cell = size_t(ntime) * es + size_t(nstat) * nout * out_es;
  const int64_t cells = std::max<int64_t>(1, static_cast<int64_t>(budget / (2 * per_cell)));
  const int64_t nb = std::min(cells, ninner);
  const int64_t ko = nb == ninner ? std::max<int64_t>(1, std::min(cells / ninner, nouter)) : 1;
  auto al = [](size_t b) { return (b + 255) / 256 * 256; };
  const size_t b_in = al(size_t(ko) * nb * ntime * es);
  const size_t b_out = al(size_t(ko) * nb * nout * out_es);
  const size_t stage_bytes = b_in + nstat * b_out;

  StagePair stage;
  WB2_TRY(stage.alloc(stage_bytes));
  StagePipe pipe(ctx, stage.buf[0], stage.buf[1]);
  const char* xh = static_cast<const char*>(x);
  for (int64_t o0 = 0; o0 < nouter; o0 += ko) {
    const int64_t k = std::min(ko, nouter - o0);
    for (int64_t c0 = 0; c0 < ninner; c0 += nb) {
      const int64_t n = std::min(nb, ninner - c0);
      char* in;
      WB2_TRY(pipe.next(&in));
      void* out[4] = {nullptr, nullptr, nullptr, nullptr};
      char* op = in + b_in;
      for (int s = 0; s < nout_host; ++s)
        if (out_host[s]) {
          out[s] = op;
          op += b_out;
        }
      WB2_TRY(pipe.h2d_2d(in, size_t(n) * es, xh + (size_t(o0) * ntime * ninner + c0) * es,
                          size_t(ninner) * es, size_t(n) * es, size_t(k) * ntime));
      WB2_TRY(pipe.ready());
      WB2_TRY(launch(static_cast<const void*>(in), k, n, static_cast<void* const*>(out)));
      for (int s = 0; s < nout_host; ++s) {
        if (!out_host[s]) continue;
        if (out_major)
          WB2_TRY(pipe.d2h_2d(out_host[s] + (size_t(o0) * ninner + c0) * out_es,
                              size_t(nouter) * ninner * out_es, out[s],
                              size_t(k) * n * out_es, size_t(k) * n * out_es, size_t(nout)));
        else
          WB2_TRY(pipe.d2h_2d(out_host[s] + (size_t(o0) * nout * ninner + c0) * out_es,
                              size_t(ninner) * out_es, out[s], size_t(n) * out_es,
                              size_t(n) * out_es, size_t(k) * nout));
      }
      WB2_TRY(pipe.done());
    }
  }
  return pipe.finish();
}

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

// Slab gather: wb2_slab_gather (device source) and wb2_slab_gather_host (NumPy /
// memmap source streamed in bands of output slabs).
//
//   out[s][i] = offsets[s] < 0 ? NaN : (To) src[offsets[s] + i],  i < slab
//
// The hot path of the reindexing operators (weatherbench2_b200/reindexing.py):
// an expanded climatology, a forecast on valid time and a probabilistic
// climatological forecast are each one output slab per outer index, copied
// from one source slab or filled with NaN.  Source and output are float32 or
// float64 in any combination; float64 -> float32 rounds to nearest, as NumPy's
// astype does, so the result is bit-exact.
//
// Two kernels, chosen from `slab`:
//   slab >= kFlatMaxSlab  slab_chunk_kernel: one CTA per (slab, chunk of
//       kChunkElems).  When some head h < 4 makes both src + off + h and
//       out + s * slab + h 16-byte aligned, the chunk moves groups of four
//       elements with 16-byte loads and stores (two of each for float64) and
//       the <= 3 head and tail elements one by one; otherwise it copies
//       element by element.  The choice is per slab and uniform in the CTA.
//   slab <  kFlatMaxSlab  slab_flat_kernel: the output flattened, each CTA
//       kFlatPer * kSgThreads consecutive output elements, so a CTA spans many
//       slabs (a station series has slab = 1, a 64 x 32 grid slab = 2048) and
//       every warp store is contiguous.
// All indexing is int64.  Every table is validated on the host before any
// launch; an invalid one never reaches the device.
#include <math_constants.h>

#include <algorithm>
#include <climits>
#include <vector>

#include "stage.cuh"

namespace wb2 {

constexpr int kSgThreads = 256;
constexpr int kVec = 4;                                      // elements per vector group
constexpr int kUnroll = 4;                                   // groups per thread
constexpr int64_t kChunkElems = int64_t(kSgThreads) * kVec * kUnroll;  // per CTA
constexpr int kScalarPer = kVec * kUnroll;                   // scalar path, per thread
constexpr int kFlatPer = 8;                                  // flat path, per thread
constexpr int64_t kFlatMaxSlab = 4096;
// host entry: runs of at least this many bytes are copied straight from the
// source; shorter ones are packed on the host and copied together
constexpr size_t kDirectRunBytes = 256 << 10;

__device__ __forceinline__ void load4(const float* p, float v[4]) {
  const float4 r = ldg_stream(reinterpret_cast<const float4*>(p));
  v[0] = r.x;
  v[1] = r.y;
  v[2] = r.z;
  v[3] = r.w;
}
__device__ __forceinline__ void load4(const double* p, double v[4]) {
  const double2 a = ldg_stream(reinterpret_cast<const double2*>(p));
  const double2 b = ldg_stream(reinterpret_cast<const double2*>(p) + 1);
  v[0] = a.x;
  v[1] = a.y;
  v[2] = b.x;
  v[3] = b.y;
}
__device__ __forceinline__ void store4(float* p, const float v[4]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}
__device__ __forceinline__ void store4(double* p, const double v[4]) {
  reinterpret_cast<double2*>(p)[0] = make_double2(v[0], v[1]);
  reinterpret_cast<double2*>(p)[1] = make_double2(v[2], v[3]);
}

__device__ __forceinline__ bool aligned16(const void* p) {
  return (reinterpret_cast<uintptr_t>(p) & 15) == 0;
}

template <typename Ti, typename To>
__global__ void __launch_bounds__(kSgThreads)
    slab_chunk_kernel(const Ti* __restrict__ src, To* __restrict__ out,
                      const int64_t* __restrict__ off, int64_t slab, int64_t nchunk) {
  const int64_t b = blockIdx.x;
  const int64_t s = b / nchunk, c = b - s * nchunk;
  const int64_t o = off[s];
  const bool fill = o < 0;
  const Ti* in = src + (fill ? 0 : o);
  To* dst = out + s * slab;
  const To qnan = To(CUDART_NAN);
  int h = -1;  // first element at which source and output are both 16-B aligned
#pragma unroll
  for (int k = kVec - 1; k >= 0; --k)
    if (aligned16(dst + k) && (fill || aligned16(in + k))) h = k;
  if (h >= 0 && h < slab) {
    const int64_t nv = (slab - h) / kVec;
    const int64_t g0 = c * (int64_t(kSgThreads) * kUnroll) + threadIdx.x;
    Ti v[kUnroll][kVec];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const int64_t g = g0 + int64_t(u) * kSgThreads;
      if (g < nv && !fill) load4(in + h + g * kVec, v[u]);
    }
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const int64_t g = g0 + int64_t(u) * kSgThreads;
      if (g < nv) {
        To w[kVec];
#pragma unroll
        for (int k = 0; k < kVec; ++k) w[k] = fill ? qnan : To(v[u][k]);
        store4(dst + h + g * kVec, w);
      }
    }
    if (c == 0 && threadIdx.x < kVec) {  // head [0, h) and tail past the groups
      const int64_t hi = threadIdx.x, ti = h + nv * kVec + threadIdx.x;
      if (hi < h) dst[hi] = fill ? qnan : To(in[hi]);
      if (ti < slab) dst[ti] = fill ? qnan : To(in[ti]);
    }
    return;
  }
  const int64_t e0 = c * kChunkElems + threadIdx.x;
  Ti v[kScalarPer];
#pragma unroll
  for (int u = 0; u < kScalarPer; ++u) {
    const int64_t i = e0 + int64_t(u) * kSgThreads;
    if (i < slab && !fill) v[u] = ldg_stream(in + i);
  }
#pragma unroll
  for (int u = 0; u < kScalarPer; ++u) {
    const int64_t i = e0 + int64_t(u) * kSgThreads;
    if (i < slab) dst[i] = fill ? qnan : To(v[u]);
  }
}

template <typename Ti, typename To>
__global__ void __launch_bounds__(kSgThreads)
    slab_flat_kernel(const Ti* __restrict__ src, To* __restrict__ out,
                     const int64_t* __restrict__ off, int64_t slab, int64_t total,
                     double inv_slab) {
  const int64_t e0 = int64_t(blockIdx.x) * (int64_t(kSgThreads) * kFlatPer) + threadIdx.x;
  const To qnan = To(CUDART_NAN);
  Ti v[kFlatPer];
  bool fill[kFlatPer];
#pragma unroll
  for (int u = 0; u < kFlatPer; ++u) {
    const int64_t e = e0 + int64_t(u) * kSgThreads;
    fill[u] = true;
    if (e < total) {
      // e / slab without a 64-bit division (a call with a stack frame): the
      // float64 quotient is within one of it while total < 2^52
      int64_t s = __double2ll_rz(double(e) * inv_slab);
      int64_t i = e - s * slab;
      if (i < 0) {
        --s;
        i += slab;
      } else if (i >= slab) {
        ++s;
        i -= slab;
      }
      const int64_t o = off[s];
      fill[u] = o < 0;
      if (o >= 0) v[u] = ldg_stream(src + o + i);
    }
  }
#pragma unroll
  for (int u = 0; u < kFlatPer; ++u) {
    const int64_t e = e0 + int64_t(u) * kSgThreads;
    if (e < total) out[e] = fill[u] ? qnan : To(v[u]);
  }
}

template <typename Ti, typename To>
static int sg_launch_t(wb2_ctx* ctx, const void* src, void* out, const int64_t* d_off,
                       int64_t slab, int64_t nslab) {
  const Ti* x = static_cast<const Ti*>(src);
  To* y = static_cast<To*>(out);
  if (slab < kFlatMaxSlab) {
    const int64_t total = slab * nslab;
    const int64_t per = int64_t(kSgThreads) * kFlatPer;
    const int64_t nblk = (total + per - 1) / per;
    WB2_REQUIRE(nblk <= INT_MAX && total < (int64_t(1) << 52),
                "nslab = %lld is too many for the slab gather's grid",
                static_cast<long long>(nslab));
    slab_flat_kernel<Ti, To><<<static_cast<unsigned>(nblk), kSgThreads, 0, ctx->stream>>>(
        x, y, d_off, slab, total, 1.0 / double(slab));
  } else {
    const int64_t nchunk = (slab + kChunkElems - 1) / kChunkElems;
    WB2_REQUIRE(nslab <= INT_MAX / nchunk,
                "nslab = %lld slabs of %lld are too many for the slab gather's grid",
                static_cast<long long>(nslab), static_cast<long long>(slab));
    slab_chunk_kernel<Ti, To>
        <<<static_cast<unsigned>(nslab * nchunk), kSgThreads, 0, ctx->stream>>>(x, y, d_off,
                                                                                slab, nchunk);
  }
  WB2_CUDA_TRY(cudaGetLastError());
  ctx->launches += 1;
  return WB2_OK;
}

static int sg_launch(wb2_ctx* ctx, int src_dtype, int out_dtype, const void* src, void* out,
                     const int64_t* d_off, int64_t slab, int64_t nslab) {
  if (src_dtype == WB2_F32)
    return out_dtype == WB2_F32
               ? sg_launch_t<float, float>(ctx, src, out, d_off, slab, nslab)
               : sg_launch_t<float, double>(ctx, src, out, d_off, slab, nslab);
  return out_dtype == WB2_F32 ? sg_launch_t<double, float>(ctx, src, out, d_off, slab, nslab)
                              : sg_launch_t<double, double>(ctx, src, out, d_off, slab, nslab);
}

static int sg_validate(const void* src, int src_dtype, int64_t src_elems, int64_t slab,
                       int64_t nslab, const int64_t* offsets, const void* out, int out_dtype) {
  WB2_REQUIRE(src_dtype == WB2_F32 || src_dtype == WB2_F64,
              "src_dtype must be WB2_F32 or WB2_F64 (got %d)", src_dtype);
  WB2_REQUIRE(out_dtype == WB2_F32 || out_dtype == WB2_F64,
              "out_dtype must be WB2_F32 or WB2_F64 (got %d)", out_dtype);
  WB2_REQUIRE(src_elems >= 0, "src_elems must be >= 0 (got %lld)",
              static_cast<long long>(src_elems));
  WB2_REQUIRE(slab >= 0 && nslab >= 0, "slab and nslab must be >= 0 (got %lld, %lld)",
              static_cast<long long>(slab), static_cast<long long>(nslab));
  if (slab == 0 || nslab == 0) return WB2_OK;
  WB2_REQUIRE(nslab <= INT64_MAX / slab, "nslab * slab overflows int64");
  WB2_REQUIRE(offsets != nullptr, "offsets is NULL");
  WB2_REQUIRE(out != nullptr, "out is NULL");
  bool any = false;
  for (int64_t s = 0; s < nslab; ++s) {
    const int64_t o = offsets[s];
    if (o < 0) continue;
    any = true;
    WB2_REQUIRE(slab <= src_elems && o <= src_elems - slab,
                "offsets[%lld] = %lld: the slab [%lld, %lld) ends past src_elems = %lld",
                static_cast<long long>(s), static_cast<long long>(o),
                static_cast<long long>(o), static_cast<long long>(o) + slab,
                static_cast<long long>(src_elems));
  }
  WB2_REQUIRE(!any || src != nullptr, "src is NULL");
  return WB2_OK;
}

static size_t sg_es(int dtype) { return dtype == WB2_F32 ? 4 : 8; }
static size_t al256(size_t b) { return (b + 255) / 256 * 256; }

// Device bytes of one staging buffer for k slabs of n elements:
// [output k*n][remapped table k][packed source, at most k*n].
static size_t sg_band_bytes(int64_t k, int64_t n, size_t es_in, size_t es_out) {
  return al256(size_t(k) * n * es_out) + al256(size_t(k) * 8) + size_t(k) * n * es_in;
}

}  // namespace wb2

using namespace wb2;

extern "C" {

int wb2_slab_gather(wb2_ctx* ctx, const void* src, int src_dtype, int64_t src_elems,
                    int64_t slab, int64_t nslab, const int64_t* offsets, void* out,
                    int out_dtype) {
  WB2_NVTX("wb2_slab_gather");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_TRY(sg_validate(src, src_dtype, src_elems, slab, nslab, offsets, out, out_dtype));
  if (slab == 0 || nslab == 0) return WB2_OK;
  DeviceGuard guard(ctx->device);
  DeviceBlock table;
  size_t o[1];
  WB2_TRY(upload_parts(ctx, {{offsets, size_t(nslab) * 8}}, &table, o));
  return sg_launch(ctx, src_dtype, out_dtype, src, out, table.at<const int64_t>(o[0]), slab,
                   nslab);
}

int wb2_slab_gather_host(wb2_ctx* ctx, const void* src, int src_dtype, int64_t src_elems,
                         int64_t slab, int64_t nslab, const int64_t* offsets, size_t budget,
                         void* out, int out_dtype) {
  WB2_NVTX("wb2_slab_gather_host");
  WB2_REQUIRE(ctx != nullptr, "ctx is NULL");
  WB2_TRY(sg_validate(src, src_dtype, src_elems, slab, nslab, offsets, out, out_dtype));
  if (slab == 0 || nslab == 0) return WB2_OK;
  const size_t es_in = sg_es(src_dtype), es_out = sg_es(out_dtype);
  const size_t half = budget / 2;
  // A band is k whole slabs, or (when one slab does not fit) a piece of n
  // elements of one slab.
  int64_t k = 1, n = slab;
  if (sg_band_bytes(1, slab, es_in, es_out) <= half) {
    const size_t per = size_t(slab) * (es_in + es_out) + 8;
    k = std::max<int64_t>(1, std::min<int64_t>(nslab, int64_t((half - std::min(half, size_t(512))) / per)));
    while (k > 1 && sg_band_bytes(k, slab, es_in, es_out) > half) --k;
  } else {
    n = int64_t(half / (es_in + es_out));
    while (n > 0 && sg_band_bytes(1, n, es_in, es_out) > half) --n;
    WB2_REQUIRE(n > 0, "budget = %zu bytes cannot hold one element in each of two buffers",
                budget);
  }
  DeviceGuard guard(ctx->device);
  const size_t b_out = al256(size_t(k) * n * es_out), b_tab = al256(size_t(k) * 8);
  StagePair stage;
  WB2_TRY(stage.alloc(sg_band_bytes(k, n, es_in, es_out)));
  StagePipe pipe(ctx, stage.buf[0], stage.buf[1]);
  const char* xh = static_cast<const char*>(src);
  char* yh = static_cast<char*>(out);
  std::vector<int64_t> table[2] = {std::vector<int64_t>(k), std::vector<int64_t>(k)};
  std::vector<int64_t> order(k);
  std::vector<char> pack;
  int cur = 0;
  for (int64_t s0 = 0; s0 < nslab; s0 += k) {
    const int64_t kb = std::min(k, nslab - s0);
    for (int64_t e0 = 0; e0 < slab; e0 += n) {
      const int64_t nb = std::min(n, slab - e0);
      char* buf;
      WB2_TRY(pipe.next(&buf));
      char* dsrc = buf + b_out + b_tab;
      int64_t* tab = table[cur].data();
      // Distinct source ranges of the band in source order; ranges that touch
      // or overlap are one run, uploaded once.
      int64_t nref = 0;
      for (int64_t j = 0; j < kb; ++j) {
        tab[j] = -1;
        if (offsets[s0 + j] >= 0) order[nref++] = j;
      }
      std::sort(order.begin(), order.begin() + nref,
                [&](int64_t a, int64_t b) { return offsets[s0 + a] < offsets[s0 + b]; });
      int64_t pos = 0, pack_at = 0;
      pack.clear();
      auto flush = [&]() -> int {
        if (!pack.empty()) WB2_TRY(pipe.h2d(dsrc + pack_at * es_in, pack.data(), pack.size()));
        pack.clear();
        pack_at = pos;
        return WB2_OK;
      };
      for (int64_t r = 0; r < nref;) {
        const int64_t start = offsets[s0 + order[r]] + e0;
        int64_t end = start + nb;
        int64_t q = r;
        for (; q < nref && offsets[s0 + order[q]] + e0 <= end; ++q) {
          end = std::max(end, offsets[s0 + order[q]] + e0 + nb);
          tab[order[q]] = pos + (offsets[s0 + order[q]] + e0 - start);
        }
        const size_t bytes = size_t(end - start) * es_in;
        const char* hp = xh + size_t(start) * es_in;
        if (bytes >= kDirectRunBytes) {
          WB2_TRY(flush());
          WB2_TRY(pipe.h2d(dsrc + pos * es_in, hp, bytes));
          pos += end - start;
          pack_at = pos;
        } else {
          pack.insert(pack.end(), hp, hp + bytes);
          pos += end - start;
        }
        r = q;
      }
      WB2_TRY(flush());
      // the table is band metadata, not source data: not counted as transfer
      WB2_CUDA_TRY(cudaMemcpyAsync(buf + b_out, tab, size_t(kb) * 8, cudaMemcpyHostToDevice,
                                   ctx->copy_stream));
      WB2_TRY(pipe.ready());
      WB2_TRY(sg_launch(ctx, src_dtype, out_dtype, dsrc, buf,
                        reinterpret_cast<const int64_t*>(buf + b_out), nb, kb));
      WB2_TRY(pipe.d2h(yh + (size_t(s0) * slab + e0) * es_out, buf, size_t(kb) * nb * es_out));
      WB2_TRY(pipe.done());
      cur ^= 1;
    }
  }
  return pipe.finish();
}

}  // extern "C"

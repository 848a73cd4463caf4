// Block-sum finalize of the region-weighted metric kernels (region_reduce.cuh).
#include "region_reduce.cuh"

namespace wb2 {

__global__ void block_sum_kernel(const double* __restrict__ partial, double* __restrict__ out,
                                 int nblk, int per_field) {
  const int64_t field = blockIdx.x;
  for (int i = threadIdx.x; i < per_field; i += blockDim.x) {
    const double* src = partial + field * int64_t(nblk) * per_field + i;
    double v = 0.0;
    for (int b = 0; b < nblk; ++b) v += src[int64_t(b) * per_field];
    out[field * per_field + i] = v;
  }
}

int launch_block_sum(wb2_ctx* ctx, const double* partial, double* out, int64_t nfield, int nblk,
                     int per_field) {
  block_sum_kernel<<<static_cast<unsigned>(nfield), 128, 0, ctx->stream>>>(partial, out, nblk,
                                                                          per_field);
  WB2_CUDA_TRY(cudaGetLastError());
  return WB2_OK;
}

}  // namespace wb2

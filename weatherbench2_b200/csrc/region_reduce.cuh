// Host side of the region-weighted spatial reduction shared by the metric
// kernels (K1 det, K2 ens, K2b ens_big, K3 energy, K7 threshold); see
// DESIGN.md section 2.  The kernels reduce a field's rows in blocks of
// `rows_per_block`, write one float64 partial block per CTA, and
// launch_block_sum adds the blocks of every field in a fixed order (no float
// atomics: the results are deterministic).  The device-side weighting (region
// application with zero_skip, skipna weight sums, CTA combine) stays written
// out in each kernel: moving it into shared inline functions, even verbatim,
// changes the generated code of the register-tight hot kernels.
#pragma once

#include <algorithm>

#include "common.cuh"

namespace wb2 {

// Uploads the weight tables of `w` through a Packer (in the order row_w,
// seg_start, seg_w, col_w) and, after commit(), fills the weight fields of a
// kernel's parameter struct.
class WeightUpload {
 public:
  WeightUpload(Packer& pk, const wb2_weights* w) : pk_(pk), w_(w) {
    const size_t R = size_t(w->nregion);
    o_rw_ = pk.add(w->row_w, R * w->nrow * sizeof(double));
    o_ss_ = pk.add(w->seg_start, size_t(w->nseg + 1) * sizeof(int32_t));
    o_sw_ = pk.add(w->seg_w, R * w->nseg * sizeof(double));
    o_cw_ = w->col_w ? pk.add(w->col_w, size_t(w->ncol) * sizeof(float)) : 0;
  }
  template <typename P>
  void bind(P& p) const {
    p.row_w = pk_.dev<double>(o_rw_);
    p.seg_start = pk_.dev<int32_t>(o_ss_);
    p.seg_w = pk_.dev<double>(o_sw_);
    p.col_w = w_->col_w ? pk_.dev<float>(o_cw_) : nullptr;
    p.cell_w = w_->cell_w;
    p.nrow = w_->nrow; p.ncol = w_->ncol; p.row_stride = w_->row_stride;
    p.nregion = w_->nregion; p.nseg = w_->nseg; p.zero_skip = w_->zero_skip;
  }

 private:
  const Packer& pk_;
  const wb2_weights* w_;
  size_t o_rw_, o_ss_, o_sw_, o_cw_;
};

// Rows per CTA and CTAs per field: `rows` rows per CTA, halved (down to
// `min_rows`) while fewer than `min_ctas` CTAs would be launched, so that
// small launches still give every SM work.
struct BlockRows {
  int rows_per_block, nblk;
};
inline BlockRows block_rows(int nrow, int64_t nfield, int rows, int min_rows, int64_t min_ctas) {
  int nblk = (nrow + rows - 1) / rows;
  while (nblk * nfield < min_ctas && rows > min_rows) {
    rows = std::max(min_rows, rows / 2);
    nblk = (nrow + rows - 1) / rows;
  }
  return {rows, nblk};
}

// K1's accumulator slot behind public stat `st` of WB2_DET_NSTAT (-1: not
// produced): the `nsum` sums, then the weight sums -- one per statistic group
// with skipna (four with a climatology), otherwise one shared by all.
constexpr int k1_slot(int st, int nsum, bool clim, bool skipna) {
  int slot = -1;
  if (st < 6) {
    if (st < nsum) slot = st;
  } else {
    const int j = st - 6;
    if (skipna) {
      if (j < (clim ? 4 : 1)) slot = nsum + j;
    } else if (clim || j == 0) {
      slot = nsum;
    }
  }
  return slot;
}

// partial [nfield][nblk][per_field] -> out [nfield][per_field], the blocks
// added in order
int launch_block_sum(wb2_ctx* ctx, const double* partial, double* out, int64_t nfield, int nblk,
                     int per_field);

}  // namespace wb2

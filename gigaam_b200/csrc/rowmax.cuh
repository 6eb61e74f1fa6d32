// The per-frame greedy score m[t] = max_c lp[t, c] of keyword spotting and of gap alignment (include/gigaam_b200.h,
// gam_ctc_spot and gam_ctc_align_long_gaps), computed by one whole warp.
#pragma once
#include <cmath>

namespace gam {

// max over row[0, V1), returned to every lane: NaN when the row holds a NaN, and + 0 so that a zero max is +0 whatever the
// order of the max.  The max is exact, so the result does not depend on the lanes' order.
__device__ __forceinline__ float warp_row_max(const float* row, int V1, int lane) {
  float mx = -INFINITY;
  int nan = 0;
  for (int c = lane; c < V1; c += 32) {
    const float x = row[c];
    mx = fmaxf(mx, x);
    nan |= isnan(x);
  }
#pragma unroll
  for (int off = 16; off; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
  if (__any_sync(0xffffffffu, nan)) mx = __int_as_float(0x7fc00000);
  return mx + 0.f;
}

}  // namespace gam

// Element and row bodies shared by the post-processing kernels.  The kernels that run one of these bodies alone
// (minmax_inverse_kernel, anomaly_score_kernel) and the one that runs both in a single pass (minmax_inverse_score_kernel) call
// the same code, so every value the fused pass writes is bit for bit what the two separate launches write.
#pragma once
#include "gb_common.cuh"

namespace gb_post {

// X -= min_; X /= scale_ on a float32 array with float64 attributes (*mn, *scale): numpy computes each in-place step in float64 and stores
// float32.  A true division, as numpy does it, not a multiplication by a reciprocal.
__device__ __forceinline__ float minmax_inverse(float p, const double* mn, const double* scale) {
  const float t = __double2float_rn(__dsub_rn((double)p, __ldg(mn)));
  return __double2float_rn(__ddiv_rn((double)t, __ldg(scale)));
}

}  // namespace gb_post

// One row of the anomaly columns, run by one warp: lane l accumulates tags l, l+32, ... in increasing order, an xor butterfly
// 16 -> 1 totals the lanes and lane 0 writes the row's totals.  YHAT_J is the row's prediction of tag j (evaluated once per
// tag).  The enclosing kernel provides: y, go / gy (the row's first element in the outputs / in y), job, r, n_out, lane, sc / ft
// (the slot's scale and feature thresholds; sc NULL: no scaled columns), agg_thr, inv = 1 / n_out and the outputs o_ts, o_tu,
// o_tots, o_totu, o_conf, o_totconf (any may be NULL).  A macro rather than a function: the body is then the same source in
// every kernel that runs it, and anomaly_score_kernel compiles to the instructions it compiled to before it was shared (a
// device function changes where the compiler resolves the pointers' address space, and with it the kernel's code).
#define GB_SCORE_ROW(T, YHAT_J)                                                     \
  do {                                                                              \
    T ss = 0, su = 0;                                                               \
    for (int j = lane; j < n_out; j += 32) {                                        \
      const T diff = (YHAT_J) - __ldg(y + gy + j);                                  \
      const T d = fabs(diff); /* +0.0 for yhat = -0.0, y = +0.0, as np.abs */       \
      if (o_tu) o_tu[go + j] = d;                                                   \
      su += d * d;                                                                  \
      if (sc) {                                                                     \
        const T e = d * __ldg(sc + j);                                              \
        if (o_ts) o_ts[go + j] = e;                                                 \
        ss += e * e;                                                                \
      }                                                                             \
      if (o_conf) o_conf[go + j] = d / __ldg(ft + j);                               \
    }                                                                               \
    for (int o = 16; o > 0; o >>= 1) {                                              \
      ss += __shfl_xor_sync(0xffffffffu, ss, o);                                    \
      su += __shfl_xor_sync(0xffffffffu, su, o);                                    \
    }                                                                               \
    if (lane == 0) {                                                                \
      if (o_tots) o_tots[job.out_row + r] = ss * inv;                               \
      if (o_totu) o_totu[job.out_row + r] = su * inv;                               \
      if (o_totconf) o_totconf[job.out_row + r] = ss * inv / __ldg(agg_thr + job.slot); \
    }                                                                               \
  } while (0)


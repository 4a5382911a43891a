// Observation normalisation (include/r2d2_b200.h, r2d2_obs_norm_merge / r2d2_obs_normalize): one transform shared by
// the replay gather, the actors' step kernel and the standalone kernel, and the Chan merge of moment blocks.
//
// A moment block is [1 + 2 O] doubles: count, mean [O], M2 [O] (sum of squared deviations from the mean).
#pragma once
#include "common.cuh"

namespace r2d2 {

// x_hat = clamp(fl(fl(x - mean) * inv_std), -c, c).  NaN passes through, as torch.clamp lets it (fminf / fmaxf would
// turn it into +-c).
__device__ __forceinline__ float obs_norm_apply(float x, float mean, float inv_std, float clip) {
  const float v = __fmul_rn(__fsub_rn(x, mean), inv_std);
  return v < -clip ? -clip : (v > clip ? clip : v);
}

// Chan's parallel merge of (nb, mb, M2b) into (na, ma, M2a) for one feature; na is not updated here (the count is
// shared by all features).  An empty side takes the other side's values unchanged.  Explicit round-to-nearest
// operations: no contraction into FMA, so the host restatement (tests/obs_norm_oracle.py) gives the same bits.
__device__ __forceinline__ void chan_merge(double na, double& ma, double& m2a, double nb, double mb, double m2b) {
  if (nb == 0.0) return;
  if (na == 0.0) { ma = mb; m2a = m2b; return; }
  const double n = __dadd_rn(na, nb);
  const double d = __dsub_rn(mb, ma);
  ma = __dadd_rn(ma, __ddiv_rn(__dmul_rn(d, nb), n));
  m2a = __dadd_rn(__dadd_rn(m2a, m2b), __ddiv_rn(__dmul_rn(__dmul_rn(__dmul_rn(d, d), na), nb), n));
}

int obs_norm_merge(double* running, const double* blocks, int W, int O, float* mean_f, float* inv_std_f,
                   cudaStream_t stream);
int obs_normalize(const float* x, float* y, long long rows, int O, const float* mean_f, const float* inv_std_f,
                  float clip, cudaStream_t stream);

}  // namespace r2d2

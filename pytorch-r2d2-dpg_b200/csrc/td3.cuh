#pragma once
#include "common.cuh"

namespace r2d2 {

// TD3's target (Fujimoto et al. 2018), off by default: target policy smoothing and the clipped double-Q minimum.
//
// Target policy smoothing: a' = clip(mu' + clip(sigma z, -c, c), -1, 1), z ~ N(0, 1) from a counter-based generator, so
// the noise is a pure function of (seed, rank, iter, element) with no generator state:
//   Philox4x32-10, key = (seed, rank), counter = (e >> 2, iter_lo, iter_hi, 0) for element e of the slice;
//   the output words (x0, x1) feed elements e % 4 in {0, 1}, (x2, x3) feed {2, 3};
//   u = (2 (x >> 9) + 1) 2^-24 (exact in fp32, in (0, 1));
//   z = sqrt(-2 ln u1) {cos, sin}(2 pi u2), cos for the even element of the pair, with precise logf / sqrtf / sincospif.
// iter is the index of the learner iteration that trains on the batch (learner.cuh Learner::critic_iters).
int target_smoothing(const float* mu, float* out, long long n, float sigma, float clip, unsigned int seed,
                     unsigned int rank, unsigned long long iter, cudaStream_t stream);
// q_next[i] = min(q_next[i], q_next2[i]) in place: the clipped double-Q bootstrap of the twin critic
int q_min(float* q_next, const float* q_next2, long long n, cudaStream_t stream);

}  // namespace r2d2

// TD3's target (td3.cuh): target policy smoothing with in-kernel Philox4x32-10 noise, and the clipped double-Q minimum.
#include "philox.cuh"
#include "td3.cuh"

namespace r2d2 {
namespace {

// one thread per group of four consecutive elements: one Philox block, two Box-Muller pairs
__global__ void __launch_bounds__(256) target_smoothing_kernel(const float* __restrict__ mu, float* __restrict__ out,
                                                               long long n, float sigma, float clip, uint32_t seed,
                                                               uint32_t rank, uint32_t iter_lo, uint32_t iter_hi) {
  const long long groups = (n + 3) >> 2;
  for (long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x; g < groups;
       g += (long long)gridDim.x * blockDim.x) {
    const Philox4 r = philox4x32_10((uint32_t)g, iter_lo, iter_hi, 0u, seed, rank);
#pragma unroll
    for (int pair = 0; pair < 2; ++pair) {
      float rad, s, c;
      box_muller(r.x[2 * pair], r.x[2 * pair + 1], rad, s, c);
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const long long e = 4 * g + 2 * pair + k;
        if (e < n) {
          const float z = __fmul_rn(rad, k ? s : c);
          const float noise = fminf(fmaxf(__fmul_rn(sigma, z), -clip), clip);
          out[e] = fminf(fmaxf(__fadd_rn(mu[e], noise), -1.0f), 1.0f);
        }
      }
    }
  }
}

__global__ void __launch_bounds__(256) q_min_kernel(float* __restrict__ q_next, const float* __restrict__ q_next2,
                                                    long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    q_next[i] = fminf(q_next[i], q_next2[i]);
}

}  // namespace

int target_smoothing(const float* mu, float* out, long long n, float sigma, float clip, unsigned int seed,
                     unsigned int rank, unsigned long long iter, cudaStream_t stream) {
  R2D2_REQUIRE(mu && out && n > 0, "target_smoothing args");
  R2D2_REQUIRE(sigma >= 0.0f && sigma <= 3.0e38f && clip > 0.0f && clip <= 3.0e38f, "sigma >= 0 and clip > 0, finite");
  const long long groups = (n + 3) >> 2;
  long long blocks = (groups + 255) / 256;
  if (blocks > num_sms() * 8) blocks = num_sms() * 8;
  target_smoothing_kernel<<<(unsigned)blocks, 256, 0, stream>>>(mu, out, n, sigma, clip, seed, rank, (uint32_t)iter,
                                                                (uint32_t)(iter >> 32));
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

int q_min(float* q_next, const float* q_next2, long long n, cudaStream_t stream) {
  R2D2_REQUIRE(q_next && q_next2 && n > 0, "q_min args");
  long long blocks = (n + 255) / 256;
  if (blocks > num_sms() * 8) blocks = num_sms() * 8;
  q_min_kernel<<<(unsigned)blocks, 256, 0, stream>>>(q_next, q_next2, n);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

}  // namespace r2d2

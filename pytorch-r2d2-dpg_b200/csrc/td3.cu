// TD3's target (td3.cuh): target policy smoothing with in-kernel Philox4x32-10 noise, and the clipped double-Q minimum.
#include "td3.cuh"

namespace r2d2 {
namespace {

// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11): ten rounds, the key bumped
// between rounds.  Known-answer vectors are checked in tests/test_cpu_td3.py (oracle) and tests/test_gpu_td3.py.
struct Philox4 { uint32_t x[4]; };

__device__ __forceinline__ Philox4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                                 uint32_t k1) {
  constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) { k0 += W0; k1 += W1; }
    const uint32_t hi0 = __umulhi(M0, c0), lo0 = M0 * c0;
    const uint32_t hi1 = __umulhi(M1, c2), lo1 = M1 * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
    c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
  }
  return Philox4{{c0, c1, c2, c3}};
}

// (0, 1), exact: the top 23 bits as an odd multiple of 2^-24
__device__ __forceinline__ float unit_open(uint32_t x) { return (float)(2u * (x >> 9) + 1u) * 0x1p-24f; }

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
      const float u1 = unit_open(r.x[2 * pair]), u2 = unit_open(r.x[2 * pair + 1]);
      const float rad = sqrtf(-2.0f * logf(u1));
      float s, c;
      sincospif(2.0f * u2, &s, &c);
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

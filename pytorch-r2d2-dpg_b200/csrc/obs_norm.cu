// Observation normalisation: the merge of per-rank moment blocks into the running statistics, and the standalone
// transform (the actor-priority chains, and the device reference of the fused routes in the gather and policy step).
#include <float.h>

#include "obs_norm.cuh"

namespace r2d2 {
namespace {

constexpr int kMergeThreads = 256;

// One CTA.  Every thread merges the W blocks into `running` in index order for its features (the counts are read by
// all threads before thread 0 rewrites running[0]), then derives the fp32 pair, each value rounded once from double.
// With no rows yet the pair is (0, 1).
__global__ void __launch_bounds__(kMergeThreads) obs_norm_merge_kernel(double* __restrict__ running,
                                                                       const double* __restrict__ blocks, int W, int O,
                                                                       float* __restrict__ mean_f,
                                                                       float* __restrict__ inv_std_f) {
  const double n0 = running[0];
  double n = n0;
  for (int w = 0; w < W; ++w) n = __dadd_rn(n, blocks[(size_t)w * (1 + 2 * O)]);
  for (int o = threadIdx.x; o < O; o += blockDim.x) {
    double na = n0, m = running[1 + o], m2 = running[1 + O + o];
    for (int w = 0; w < W; ++w) {
      const double* b = blocks + (size_t)w * (1 + 2 * O);
      chan_merge(na, m, m2, b[0], b[1 + o], b[1 + O + o]);
      na = __dadd_rn(na, b[0]);
    }
    running[1 + o] = m;
    running[1 + O + o] = m2;
    if (mean_f) {
      mean_f[o] = n > 0.0 ? __double2float_rn(m) : 0.0f;
      inv_std_f[o] = n > 0.0 ? __double2float_rn(__ddiv_rn(1.0, __dsqrt_rn(__dadd_rn(__ddiv_rn(m2, n), 1e-8)))) : 1.0f;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) running[0] = n;
}

__global__ void __launch_bounds__(256) obs_normalize_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                            long long n, int O, const float* __restrict__ mean_f,
                                                            const float* __restrict__ inv_std_f, float clip) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int o = (int)(i % O);
    y[i] = obs_norm_apply(x[i], __ldg(mean_f + o), __ldg(inv_std_f + o), clip);
  }
}

}  // namespace

int obs_norm_merge(double* running, const double* blocks, int W, int O, float* mean_f, float* inv_std_f,
                   cudaStream_t stream) {
  R2D2_REQUIRE(running && (W == 0 || blocks) && W >= 0 && O > 0, "args");
  R2D2_REQUIRE((mean_f == nullptr) == (inv_std_f == nullptr), "mean_f and inv_std_f are both given or both NULL");
  obs_norm_merge_kernel<<<1, kMergeThreads, 0, stream>>>(running, blocks, W, O, mean_f, inv_std_f);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

int obs_normalize(const float* x, float* y, long long rows, int O, const float* mean_f, const float* inv_std_f,
                  float clip, cudaStream_t stream) {
  R2D2_REQUIRE(x && y && mean_f && inv_std_f && rows >= 0 && O > 0, "args");
  R2D2_REQUIRE(clip > 0.f && clip <= FLT_MAX, "clip must be finite and > 0");
  const long long n = rows * O;
  if (n == 0) return R2D2_OK;
  long long blocks = (n + 255) / 256;
  if (blocks > num_sms() * 16) blocks = num_sms() * 16;
  obs_normalize_kernel<<<(unsigned)blocks, 256, 0, stream>>>(x, y, n, O, mean_f, inv_std_f, clip);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

}  // namespace r2d2

// Learner metrics: two reductions per iteration into the caller's ring (include/r2d2_b200.h, r2d2_learner_set_metrics).
//
//   metrics_critic_kernel  end of the critic phase: iteration, %globaltimer, the critic losses, q / target / |q - y| /
//                          q2 statistics over [L,B,A], priority and importance-weight statistics over [B], non-finite count
//   metrics_actor_kernel   actor phase, after losses[1]: the actor loss, |mu| statistics over [L,B,A], the critic's
//                          pre-clip gradient norm of this iteration's optimiser step, non-finite values of mu
//
// Both follow grad_norm_kernel's determinism rule: a fixed grid of kMetricsBlocks CTAs writes one set of double partials
// per CTA; the CTA that draws the last ticket combines them in a fixed order and writes the record.  Sums are of doubles
// in a fixed order, min / max are order-independent (fmin / fmax: a NaN is skipped there and counted in `nonfinite`),
// counts are exact.  No floating-point atomics: the same inputs write the same record bits.
#include "metrics.cuh"

#include <math.h>

namespace r2d2 {

namespace {

constexpr int MT = 256;   // threads per CTA
constexpr int MW = MT / 32;

const char* const kFieldNames[kMetricsFields] = {
    "iteration", "t_ns", "critic_loss", "critic2_loss", "actor_loss", "q_mean", "q_min", "q_max", "target_mean",
    "target_min", "target_max", "td_abs_mean", "td_abs_max", "priority_mean", "priority_max", "is_weight_min",
    "is_weight_mean", "q2_mean", "mu_abs_mean", "mu_saturated", "critic_grad_norm", "actor_grad_norm", "nonfinite"};

// field f combines by min when bit f of MinMask is set, by max when bit f of MaxMask is, else by +
template <unsigned MinMask, unsigned MaxMask>
__device__ __forceinline__ double combine(int f, double a, double b) {
  if ((MinMask >> f) & 1u) return fmin(a, b);
  if ((MaxMask >> f) & 1u) return fmax(a, b);
  return a + b;
}

// Reduces v over the grid.  Returns true in the last CTA, where out[0..NF) then holds the grid's values (all threads
// may read them); every other CTA returns false.
template <int NF, unsigned MinMask, unsigned MaxMask>
__device__ bool grid_reduce(double (&v)[NF], double* part, unsigned int* ticket, double (*s_warp)[NF], double* out) {
  __shared__ bool last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int f = 0; f < NF; ++f) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[f] = combine<MinMask, MaxMask>(f, v[f], __shfl_xor_sync(0xffffffffu, v[f], o));
    if (lane == 0) s_warp[warp][f] = v[f];
  }
  __syncthreads();
  if (threadIdx.x < NF) {
    const int f = threadIdx.x;
    double r = s_warp[0][f];
    for (int w = 1; w < MW; ++w) r = combine<MinMask, MaxMask>(f, r, s_warp[w][f]);
    part[(size_t)f * gridDim.x + blockIdx.x] = r;
  }
  __threadfence();                 // this CTA's partials are visible device-wide before its ticket is drawn
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last) return false;
  __threadfence();
  for (int f = warp; f < NF; f += MW) {     // warp w combines fields w, w + MW, ...: lanes stride the CTAs in order
    double r = ((MinMask >> f) & 1u) ? INFINITY : ((MaxMask >> f) & 1u) ? -INFINITY : 0.0;
    for (int k = lane; k < (int)gridDim.x; k += 32) r = combine<MinMask, MaxMask>(f, r, __ldcg(part + (size_t)f * gridDim.x + k));
    for (int o = 16; o > 0; o >>= 1) r = combine<MinMask, MaxMask>(f, r, __shfl_xor_sync(0xffffffffu, r, o));
    if (lane == 0) out[f] = r;
  }
  __syncthreads();
  return true;
}

__device__ __forceinline__ double nonfinite(float x) { return isfinite(x) ? 0.0 : 1.0; }

// partials: 0 sum q, 1 min q, 2 max q, 3 sum target, 4 min target, 5 max target, 6 sum |q - y|, 7 max |q - y|,
// 8 sum q2, 9 non-finite count, 10 sum priority, 11 max priority, 12 min is_weight, 13 sum is_weight
constexpr unsigned kCriticMin = (1u << 1) | (1u << 4) | (1u << 12);
constexpr unsigned kCriticMax = (1u << 2) | (1u << 5) | (1u << 7) | (1u << 11);

__global__ void __launch_bounds__(MT) metrics_critic_kernel(MetricsCriticParams p, double* part, unsigned int* ticket) {
  __shared__ double s_warp[MW][kMetricsPartials];
  __shared__ double s_out[kMetricsPartials];
  double v[kMetricsPartials] = {0.0, INFINITY, -INFINITY, 0.0, INFINITY, -INFINITY, 0.0, -INFINITY,
                                0.0, 0.0, 0.0, -INFINITY, INFINITY, 0.0};
  const long long stride = (long long)gridDim.x * MT;
  for (long long i = blockIdx.x * (long long)MT + threadIdx.x; i < p.n; i += stride) {
    const float q = p.q[i], t = p.target[i];
    const double td = fabs((double)q - (double)t);
    v[0] += q; v[1] = fmin(v[1], (double)q); v[2] = fmax(v[2], (double)q);
    v[3] += t; v[4] = fmin(v[4], (double)t); v[5] = fmax(v[5], (double)t);
    v[6] += td; v[7] = fmax(v[7], td);
    v[9] += nonfinite(q) + nonfinite(t);
    if (p.q2) {
      const float q2 = p.q2[i];
      v[8] += q2;
      v[9] += nonfinite(q2);
    }
  }
  for (long long i = blockIdx.x * (long long)MT + threadIdx.x; i < p.B; i += stride) {
    const float pr = p.priority[i], w = p.is_weight ? p.is_weight[i] : 1.0f;
    v[10] += pr; v[11] = fmax(v[11], (double)pr);
    v[12] = fmin(v[12], (double)w); v[13] += w;
  }
  if (!grid_reduce<kMetricsPartials, kCriticMin, kCriticMax>(v, part, ticket, s_warp, s_out)) return;
  if (threadIdx.x == 0) {
    unsigned long long now;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
    const double n = (double)p.n, B = (double)p.B, nan = __longlong_as_double(0x7ff8000000000000ll);
    double* r = p.rec;
    r[kMIteration] = (double)p.iter;
    r[kMTimeNs] = (double)now;
    r[kMCriticLoss] = p.losses[0];
    r[kMCritic2Loss] = p.q2 ? (double)p.losses[2] : nan;
    r[kMQMean] = s_out[0] / n; r[kMQMin] = s_out[1]; r[kMQMax] = s_out[2];
    r[kMTargetMean] = s_out[3] / n; r[kMTargetMin] = s_out[4]; r[kMTargetMax] = s_out[5];
    r[kMTdAbsMean] = s_out[6] / n; r[kMTdAbsMax] = s_out[7];
    r[kMPriorityMean] = s_out[10] / B; r[kMPriorityMax] = s_out[11];
    r[kMIsWeightMin] = s_out[12]; r[kMIsWeightMean] = s_out[13] / B;
    r[kMQ2Mean] = p.q2 ? s_out[8] / n : nan;
    r[kMNonfinite] = s_out[9];
    // the actor phase's fields: stale values of the slot's previous iteration never show
    r[kMActorLoss] = nan; r[kMMuAbsMean] = nan; r[kMMuSaturated] = nan; r[kMCriticGradNorm] = nan;
    r[kMActorGradNorm] = nan;
    *ticket = 0u;
  }
}

// partials: 0 sum |mu|, 1 count |mu| >= 0.99, 2 non-finite count (all sums)
__global__ void __launch_bounds__(MT) metrics_actor_kernel(MetricsActorParams p, double* part, unsigned int* ticket) {
  __shared__ double s_warp[MW][3];
  __shared__ double s_out[3];
  double v[3] = {0.0, 0.0, 0.0};
  for (long long i = blockIdx.x * (long long)MT + threadIdx.x; i < p.n; i += (long long)gridDim.x * MT) {
    const float a = fabsf(p.mu[i]);
    v[0] += a;
    v[1] += a >= 0.99f ? 1.0 : 0.0;
    v[2] += nonfinite(a);
  }
  if (!grid_reduce<3, 0u, 0u>(v, part, ticket, s_warp, s_out)) return;
  if (threadIdx.x == 0) {
    const double n = (double)p.n;
    double* r = p.rec;
    r[kMActorLoss] = p.losses[1];
    r[kMMuAbsMean] = s_out[0] / n;
    r[kMMuSaturated] = s_out[1] / n;
    r[kMCriticGradNorm] = *p.critic_norm;
    r[kMNonfinite] += s_out[2];
    *ticket = 0u;
  }
}

}  // namespace

const char* metrics_field_name(int i) { return i >= 0 && i < kMetricsFields ? kFieldNames[i] : nullptr; }

int metrics_critic(const MetricsCriticParams& p, double* part, unsigned int* ticket, cudaStream_t stream) {
  R2D2_REQUIRE(p.q && p.target && p.priority && p.losses && p.rec && part && ticket && p.n > 0 && p.B > 0,
               "metrics_critic args");
  metrics_critic_kernel<<<kMetricsBlocks, MT, 0, stream>>>(p, part, ticket);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

int metrics_actor(const MetricsActorParams& p, double* part, unsigned int* ticket, cudaStream_t stream) {
  R2D2_REQUIRE(p.mu && p.losses && p.critic_norm && p.rec && part && ticket && p.n > 0, "metrics_actor args");
  metrics_actor_kernel<<<kMetricsBlocks, MT, 0, stream>>>(p, part, ticket);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

}  // namespace r2d2

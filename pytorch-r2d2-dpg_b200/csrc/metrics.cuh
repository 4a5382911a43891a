// Learner metrics (include/r2d2_b200.h, r2d2_learner_set_metrics): one double[kMetricsFields] record per learner
// iteration, reduced on the device in the learner's stream into a caller-owned ring.
#pragma once
#include "common.cuh"

namespace r2d2 {

constexpr int kMetricsFields = 23;
constexpr int kMetricsBlocks = 256;      // fixed grid of both reductions: same inputs, same bits
constexpr int kMetricsPartials = 14;     // per-CTA partial values of the critic kernel (the actor kernel uses 3)

// record field indices (names: metrics_field_name)
enum MetricsField {
  kMIteration = 0, kMTimeNs, kMCriticLoss, kMCritic2Loss, kMActorLoss, kMQMean, kMQMin, kMQMax, kMTargetMean,
  kMTargetMin, kMTargetMax, kMTdAbsMean, kMTdAbsMax, kMPriorityMean, kMPriorityMax, kMIsWeightMin, kMIsWeightMean,
  kMQ2Mean, kMMuAbsMean, kMMuSaturated, kMCriticGradNorm, kMActorGradNorm, kMNonfinite
};

const char* metrics_field_name(int i);   // NULL outside [0, kMetricsFields)

struct MetricsCriticParams {
  const float *q, *target, *q2, *priority, *is_weight, *losses;   // q2 / is_weight may be NULL (twin off / weighting off)
  long long n;   // L * B * A
  int B;
  long long iter;
  double* rec;   // the iteration's record
};

struct MetricsActorParams {
  const float *mu, *losses, *critic_norm;
  long long n;
  double* rec;
};

// One launch each.  part: kMetricsBlocks * kMetricsPartials doubles; ticket: one zeroed word the kernels leave zeroed.
int metrics_critic(const MetricsCriticParams& p, double* part, unsigned int* ticket, cudaStream_t stream);
int metrics_actor(const MetricsActorParams& p, double* part, unsigned int* ticket, cudaStream_t stream);

}  // namespace r2d2

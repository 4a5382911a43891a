#pragma once
#include "common.cuh"

namespace r2d2 {

// n-step target and priority options (include/r2d2_b200.h: R2D2_RESCALE_*, R2D2_PRIORITY_*)
constexpr int kRescaleReference = 0;    // y = h0(R + gamma^n (1-d) Q'), h0(x) = sign(x)(sqrt(|x|+1) - 1)  (utils.py:20-21)
constexpr int kRescaleInvertible = 1;   // y = h_eps(R + gamma^n (1-d) h_eps^-1(Q')), h_eps = h0 + eps x  (R2D2)
constexpr int kPrioritySquared = 0;     // priority over the squared TD errors td_sq  (utils.py:17-18)
constexpr int kPriorityAbs = 1;         // priority over their roots sqrt(td_sq): |delta| at A = 1  (R2D2)
struct TdOptions {
  int rescaling = kRescaleReference;
  float eps = 0.f;                 // h_eps's eps in [0, 1]; the reference rescaling ignores it
  int priority_metric = kPrioritySquared;
};
// R2D2_OK, or R2D2_ERR_ARG for an unknown mode / metric or (invertible only) an eps outside [0, 1], NaN included
int check_td_options(const TdOptions& opt);

struct TdPriorityParams {
  const float* q = nullptr;        // [L,B,A] online critic on (o_t, a_t), t in [Bn, Bn+L)      learner.py:105
  const float* q_next = nullptr;   // [L,B,A] target critic on (o_{t+n}, target_actor(o_{t+n}))  learner.py:106
  const float* rew = nullptr;      // [T',B] rewards, already n-step pre-summed by the actor     actor.py:74-76
  const float* term = nullptr;     // [T',B] terminal flags; row t+n-1 gates the bootstrap       learner.py:107
  float* target = nullptr;         // [L,B,A] h(R + gamma^n (1-d) Q'), or h_eps(R + gamma^n (1-d) h_eps^-1(Q'))  (optional)
  float* dq = nullptr;             // [L,B,A] d critic_loss / d q = 2 (q - y) / (L*B*A)  (optional)
  float* td_sq = nullptr;          // [L,B] mean over A of squared TD (optional)
  float* priority = nullptr;       // [B] eta*max + (1-eta)*mean over the [b:-1:B] slice of td_sq, or of sqrt(td_sq)
                                   // under kPriorityAbs (optional)
  float* loss_sum = nullptr;       // scalar: MSE-mean critic loss (zeroed by the call, optional)
  const float* is_weight = nullptr; // [B] importance weights w_b (optional): loss = sum w_b td_sq / (L*B), dq scaled by
                                    // w_b; td_sq and priority stay unweighted.  NULL: every w_b = 1, same bits
  int L = 0, B = 0, A = 0, burn_in = 0, n_step = 0;
  float gamma_n = 0.f;             // gamma ** n_step
  float eta = 0.9f;
  float eps = 0.f;                 // set by td_priority from TdOptions.  It sits in what was the struct's tail padding,
                                   // so the size and every other offset are unchanged and the default kernels, which
                                   // never read it, compile as before
};

// The mode and the metric pick the kernel instantiations; only eps reaches the kernels (p.eps is overwritten)
int td_priority(const TdPriorityParams& p, cudaStream_t stream, const TdOptions& opt = TdOptions());
// actor-side next rows (actor.py:74-107), batched over episodes: raw / out [T,B] time-major, n_rows[b] = rows of episode b
// incl. its n_step pad rows; q [T-n_step.., B, A] online critic, q_next [T,B,A] target critic on target-actor actions
int nstep_rewards(const float* raw, const int* n_rows, int T, int B, int n_step, float gamma, float* out, cudaStream_t stream);
int actor_priorities(const float* q, const float* q_next, const float* rew, const float* term, const int* n_rows, int B,
                     int A, int burn_in, int learning, int n_step, float gamma, float eta, int p_max, float* prio,
                     cudaStream_t stream, const TdOptions& opt = TdOptions());
// out[n] += sum_m x[m,n] (and out2 if given); accumulates into pre-zeroed buffers
int colsum(const float* x, long long ld, int M, int N, float* out, float* out2, cudaStream_t stream);
int add_vec(const float* a, const float* b, float* out, int n, cudaStream_t stream);
int mul_dtanh(const float* d_out, const float* out, float* d_pre, long long n, cudaStream_t stream);
// Adam on a flat buffer (grad * grad_scale).  clip_coef (device scalar from grad_norm, optional) multiplies the
// gradient first; target (optional) receives the Polyak update target = target (1 - tau) + param' tau in the same pass.
int adam_step(float* param, const float* grad, float* m, float* v, long long n, int step, float lr, float beta1,
              float beta2, float eps, float grad_scale, cudaStream_t stream, const float* clip_coef = nullptr,
              float* target = nullptr, float tau = 1.0f);
// *norm = ||grad * grad_scale||_2 and *coef = min(1, max_norm / (*norm + 1e-6)), one launch of kGradNormBlocks CTAs.
// partials: kGradNormBlocks doubles; ticket: one zeroed word the kernel leaves zeroed.  One launch at a time per ticket.
constexpr int kGradNormBlocks = 512;
int grad_norm(const float* grad, long long n, float grad_scale, float max_norm, double* partials, unsigned int* ticket,
              float* norm, float* coef, cudaStream_t stream);
int fill_f32(float* x, long long n, float value, cudaStream_t stream);
int scaled_sum(const float* x, long long n, float scale, float* out, cudaStream_t stream);

// Deterministic accumulation.  A kernel that would add many partial results into one place writes them instead into
// slices of a scratch buffer (grow-only, one per device and stream, valid until the next call on the same stream), and
// add_partials adds the slices in slice order, so that every run sums in the same order and gets the same bits:
//   dst[r * ld_dst + c] += sum_{s < slices} part[(s * rows + r) * cols + c]   (and the same sum into dst2 if given)
int partials_scratch(size_t floats, cudaStream_t stream, float** out);
int add_partials(const float* part, int slices, int rows, int cols, float* dst, long long ld_dst, float* dst2,
                 cudaStream_t stream);

}  // namespace r2d2

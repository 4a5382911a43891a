#pragma once
#include "common.cuh"
#include "elementwise.cuh"
#include "metrics.cuh"
#include "net.cuh"
#include "peer.cuh"

namespace r2d2 {

struct Learner {
  r2d2_learner_config cfg;
  NetShape actor_sh, critic_sh;
  int rows = 0;            // T' = burn_in + learning + n_step
  int step = 0;            // completed learner iterations (learner.py:82)
  int launches_phase[3] = {0, 0, 0};
  // side stream for work that depends on the batch and the weights only (the input projections of the online critic
  // chain and of the actor's DPG chain): it fills the SMs the persistent scans of the target chains leave idle
  cudaStream_t side = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_c1_inputs = nullptr, ev_a1_inputs = nullptr;
  bool overlap_inputs = false;
  bool overlap_actor_inputs = true;  // off while the caller defers the actor's optimiser step behind the next critic phase
  bool a1_inputs_pending = false;    // a1's input projection of this iteration was issued on the side stream
  bool actor_forward_done = false;   // learner_actor_forward already ran for the current iteration
  int launches_actor_forward = 0;
  // second learner-owned stream for whole chains that run beside the learner stream's (single GPU,
  // overlap_inputs on; learner.cu, learner_critic_phase): the actor's forward chain under the online critic's, the
  // critic BPTT under the next batch's target chains.  ev_aux_done: the last aux work issued; the actor phase joins it.
  // ev_q_next_read: the twin's TD on aux has read q_next, which the next target phase overwrites.
  cudaStream_t aux = nullptr;
  cudaEvent_t ev_aux_fork = nullptr, ev_aux_done = nullptr, ev_q_next_read = nullptr;
  bool aux_pending = false;          // ev_aux_done is recorded and the actor phase has not joined it yet
  bool q_next_pending = false;       // ev_q_next_read is recorded and no target phase has waited for it yet
  bool concurrent_chains() const { return aux && overlap_actor_inputs && !peer; }
  float* arena = nullptr;
  size_t arena_floats = 0;
  // batch (filled by replay_sample or by the caller).  Two slots: while the phases of iteration i still read slot s, the
  // caller may fill slot 1-s with batch i+1 and run its target chains early (learner_target_phase) - they read the
  // target nets only, so they are the independent work between "critic gradients complete" and "sums needed" of the
  // data-parallel gradient exchange.  obs .. leaf_idx below always point into slots[cur_slot].
  struct BatchSlot {
    float *obs = nullptr, *act = nullptr, *rew = nullptr, *term = nullptr, *states = nullptr, *uniforms = nullptr;
    long long* leaf_idx = nullptr;
    float* is_weight = nullptr;   // [B] importance weights of the batch (r2d2_replay_sample_weighted), 1 by default
  } slots[2];
  int cur_slot = 0;
  int targets_slot = -1;        // slot whose target-chain outputs (q_next) are current; -1: none
  int c1_inputs_slot = -1;      // slot whose online-critic input projection is in flight / done on the side stream
  int launches_target = 0;      // launches of the last learner_target_phase
  bool target_phase_standalone = false;
  float *obs = nullptr, *act = nullptr, *rew = nullptr, *term = nullptr, *states = nullptr, *uniforms = nullptr;
  long long* leaf_idx = nullptr;
  float* is_weight = nullptr;
  bool importance_weighting = false;   // the TD kernels read is_weight (off: NULL, the unweighted loss)
  // optimiser step: Polyak weight of the target update (1: the hard copy) and the per-net global gradient-norm bound
  // (0: no clipping).  optim = [critic N, actor N, critic coef, actor coef] of the last step; norm_part / norm_ticket:
  // grad_norm's partials and tickets, one set per net
  float target_tau = 1.0f;
  float grad_clip = 0.0f;
  float* optim = nullptr;
  unsigned int* norm_ticket = nullptr;
  double* norm_part = nullptr;
  // n-step target and priority options of the TD kernels (elementwise.cuh TdOptions): the reference's by default.  q_next
  // is the target critic's raw output in every mode (h_eps^-1 runs inside the TD kernel), so they may change between
  // any two iterations
  int rescaling = kRescaleReference;
  float rescaling_eps = 0.0f;
  int priority_metric = kPrioritySquared;
  // TD3's target (td3.cuh), off by default.  twin: a create-time choice - every cfg.critic_* block holds 2 P' floats
  // [critic 1 | pad | critic 2 | pad], P = critic_sh.param_count() and P' = P rounded up to 64 floats, so that critic 2's
  // matrices sit at the same 256-byte alignment as critic 1's (the GEMM kernels load them with vector accesses); the
  // padding stays zero.  Critic 1 is the reference's critic with its stored state, critic 2 and its target start from
  // the zero state.  target_noise > 0: smoothing of the target actor's actions, keyed on (noise_seed, noise_rank) and
  // critic_iters.
  bool twin = false;
  float target_noise = 0.0f, target_noise_clip = 0.5f;
  unsigned int noise_seed = 0, noise_rank = 0;
  // critic phases run so far: the index of the iteration that trains on the batch a target phase prepares (a target
  // phase run ahead after critic phase i sees i + 1, one inside critic phase i sees i); r2d2_learner_set_step_count sets it
  long long critic_iters = 0;
  size_t twin_floats = 0;   // arena floats carved for the twin (0 without it)
  size_t critic_stride() const { return twin ? (critic_sh.param_count() + 63) & ~(size_t)63 : critic_sh.param_count(); }
  size_t critic_block() const { return critic_stride() * (twin ? 2 : 1); }
  // intermediates / results
  float *act_tc = nullptr, *q = nullptr, *q_next = nullptr, *target = nullptr, *dq = nullptr, *mu = nullptr,
        *q_pi = nullptr, *dq_pi = nullptr, *dpre_actor = nullptr, *td_sq = nullptr, *priority = nullptr,
        *losses = nullptr;
  ChainWs ws_ta, ws_tc, ws_c1, ws_a1, ws_c2;
  // twin only: target critic 2 / online critic 2 chains, and critic 2's q_next, q, dq and td_sq (scratch)
  ChainWs ws_tc_2, ws_c1_2;
  float *q_next2 = nullptr, *q2 = nullptr, *dq2 = nullptr, *td_sq2 = nullptr;
  // data-parallel learner: gradient blocks live in a peer-mapped buffer and are summed by peer.cu's kernels in this
  // learner's own stream (null: single GPU, or the caller reduces cfg.*_grads itself between the phases)
  PeerExchange* peer = nullptr;
  // learner metrics (metrics.cuh), off while metrics_ring is null: the caller's ring of metrics_slots records of
  // kMetricsFields doubles followed by metrics_slots floats of actor gradient norms (r2d2_learner_set_metrics).  The
  // kernels' partials and ticket live in metrics_part, the learner's own allocation made by the first set call, so that
  // the arena and every offset in it stay as they are.  metrics_iter: the iteration of the last critic phase.
  double* metrics_ring = nullptr;
  int metrics_slots = 0;
  double* metrics_part = nullptr;
  unsigned int* metrics_ticket = nullptr;
  long long metrics_iter = 0;
  bool critic_phase_ran = false;
  double* metrics_record(long long iter) const { return metrics_ring + (size_t)(iter % metrics_slots) * kMetricsFields; }
  float* metrics_actor_norms() const {
    return reinterpret_cast<float*>(metrics_ring + (size_t)metrics_slots * kMetricsFields);
  }
  const float* optimiser_grads(int block) const {
    return peer ? peer->sums(block) : (block == kPeerCritic ? cfg.critic_grads : cfg.actor_grads);
  }
};

int learner_create(Learner** out, const r2d2_learner_config* cfg, bool twin_critic = false);
int learner_destroy(Learner* l);
int learner_select_batch(Learner* l, int slot);
// target chains of the batch in `slot` (learner.py:87,94-95,106): q_next for the next learner_critic_phase on that slot.
// Reads the target nets and the batch only.  learner_critic_phase runs it itself when the current slot has none.
int learner_target_phase(Learner* l, int slot, cudaStream_t stream);
// forget a target phase that ran ahead (the caller is about to overwrite that batch)
int learner_discard_prefetch(Learner* l, cudaStream_t stream);
int learner_critic_phase(Learner* l, cudaStream_t stream);
int learner_actor_forward(Learner* l, cudaStream_t stream);
int learner_actor_phase(Learner* l, float grad_scale, cudaStream_t stream);
int learner_finish_phase(Learner* l, float grad_scale, cudaStream_t stream);
// peer_bases[k] = rank k's exchange buffer (peer_layout(...).bytes, zeroed, mapped into this process); moves the
// learner's gradient blocks into peer_bases[rank]
int learner_attach_peers(Learner* l, int rank, int world, void* const* peer_bases);
// ring: r2d2_metrics_ring_bytes(slots) of device memory (8-byte aligned), or null for off; before the first critic phase
int learner_set_metrics(Learner* l, void* ring, int slots);

}  // namespace r2d2

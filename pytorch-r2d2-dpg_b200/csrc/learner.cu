// Learner iteration engine: learner.py:84-139 (sample excluded - see replay.cu) as three phases so a
// data-parallel caller can all-reduce the flat gradient buffers between them (NCCL lives in the host code).
//
//   phase 1  target_actor chain  -> target_critic chain -> online critic chain -> fused TD/priority
//            kernel -> critic BPTT                                          (learner.py:86-113)
//   phase 2  critic Adam; actor chain from the zero state with two cell steps per row; critic on the
//            actor's actions with the post-step weights; dgrad through the critic; actor BPTT
//                                                                             (learner.py:114-127)
//   phase 3  actor Adam; hard target update every `target_update_interval` steps (learner.py:128-132)
//
// Optional optimiser extras (off by default): global gradient-norm clipping per net (a norm kernel before each Adam) and
// a Polyak target update (target_tau < 1) on the same iterations as the hard copy, fused into the Adam launches: the
// critic's target in phase 2, the actor's in phase 3.
//
// TD3's target (off by default, td3.cuh): with target noise the target actor's actions for the bootstrap rows are
// smoothed in place right after its head; with the twin critic a second target critic (zero state) runs on the same
// actions and q_next becomes the elementwise minimum, and in phase 1 a second online critic (zero state) runs its own
// TD against the same y and its own BPTT into the second half of the critic gradient block.  Critic 1 keeps every other
// role: the DPG loss of phase 2, the priorities, td_sq and the target written out.
//
// Learner metrics (off by default, metrics.cuh): with a ring set, one reduction kernel at the end of phase 1 and one after
// the actor loss in phase 2 write the iteration's record, the norm kernel runs before each Adam even without clipping, and
// phase 3 copies the actor's norm into the ring.  Off, none of it is issued.
//
// Concurrent chains (one GPU, R2D2_OVERLAP_INPUTS not 0): phase 1 runs the actor's forward chain of phase 2, and its own
// work after the TD kernels, on a second learner-owned stream (aux) beside the learner stream's chains; phase 2 joins
// it before the critic's Adam.  Same kernels, same bits; learner_critic_phase lists the shared buffers.
//
// The actor burn-in of learner.py:92 is skipped: its state is discarded at learner.py:117 before any use.
#include "learner.cuh"

#include <cmath>
#include <stdlib.h>

#include "elementwise.cuh"
#include "gemm.cuh"
#include "lstm_scan.cuh"
#include "td3.cuh"

namespace r2d2 {

static size_t align64(size_t n) { return (n + 63) & ~(size_t)63; }

int learner_create(Learner** out, const r2d2_learner_config* cfg, bool twin_critic) {
  R2D2_REQUIRE(out && cfg, "null");
  R2D2_REQUIRE(cfg->obs_size > 0 && cfg->n_actions > 0 && cfg->hidden > 0 && cfg->hidden % 4 == 0, "sizes");
  R2D2_REQUIRE(cfg->batch > 0 && cfg->burn_in >= 0 && cfg->learning > 0 && cfg->n_step > 0, "window");
  R2D2_REQUIRE(cfg->learning >= 2, "learning >= 2: the [b:-1:B] priority series of the last batch element drops its "
                                   "last TD step, so a one-step window leaves it empty");
  R2D2_REQUIRE(cfg->actor_params && cfg->critic_params && cfg->target_actor_params && cfg->target_critic_params,
               "parameter buffers");
  R2D2_REQUIRE(cfg->actor_grads && cfg->critic_grads && cfg->actor_exp_avg && cfg->actor_exp_avg_sq &&
                   cfg->critic_exp_avg && cfg->critic_exp_avg_sq, "gradient / Adam buffers");
  Learner* l = new Learner();
  l->cfg = *cfg;
  l->actor_sh = NetShape{cfg->obs_size, cfg->n_actions, cfg->hidden, false};
  l->critic_sh = NetShape{cfg->obs_size, cfg->n_actions, cfg->hidden, true};
  const int B = cfg->batch, Bn = cfg->burn_in, L = cfg->learning, n = cfg->n_step;
  const int O = cfg->obs_size, A = cfg->n_actions, H = cfg->hidden;
  const int Tt = Bn + n + L, Tc = Bn + L, Tw = Bn + L + n;
  l->rows = Tw;
  // one allocation, carved
  size_t total = 0;
  const size_t n_obs = align64((size_t)Tw * B * O), n_act = align64((size_t)Tw * B * A), n_rt = align64((size_t)Tw * B);
  const size_t n_states = align64((size_t)8 * B * H), n_lba = align64((size_t)L * B * A);
  const size_t n_acttc = align64((size_t)Tt * B * A);
  total += 2 * (n_obs + n_act + 2 * n_rt + n_states + align64(B) /*uniforms*/ + align64(2 * (size_t)B) /*leaf idx (int64)*/);
  total += n_acttc + 8 * n_lba + align64((size_t)L * B) + align64(B) + 64;
  const size_t ws_ta = ChainWs::floats(l->actor_sh, Tt, B, 1), ws_tc = ChainWs::floats(l->critic_sh, Tt, B, 1);
  const size_t ws_c1 = ChainWs::floats(l->critic_sh, Tc, B, 1), ws_a1 = ChainWs::floats(l->actor_sh, L, B, 2);
  const size_t ws_c2 = ChainWs::floats(l->critic_sh, L, B, 1);
  total += ws_ta + ws_tc + ws_c1 + ws_a1 + ws_c2;
  total += 2 * align64(B);   // importance weights of the two slots, carved last: the buffers above keep their offsets
  total += align64(8) + align64(4 * (size_t)kGradNormBlocks);   // optimiser scalars + tickets, norm partials (2 x double)
  // twin critic: carved last, only when on, so the default arena and every offset above are unchanged
  l->twin = twin_critic;
  if (twin_critic) {
    // target / online critic 2 chains, q_next2 / q2 / dq2, td_sq2
    l->twin_floats = align64(ws_tc) + align64(ws_c1) + 3 * n_lba + align64((size_t)L * B);
    total += l->twin_floats;
  }
  R2D2_CUDA_TRY(cudaMalloc(&l->arena, total * sizeof(float)));
  R2D2_CUDA_TRY(cudaMemset(l->arena, 0, total * sizeof(float)));
  l->arena_floats = total;
  float* p = l->arena;
  auto take = [&](size_t nfl) { float* r = p; p += align64(nfl); return r; };
  for (auto& b : l->slots) {
    b.obs = take(n_obs); b.act = take(n_act); b.rew = take(n_rt); b.term = take(n_rt);
    b.states = take(n_states); b.uniforms = take(B);
    b.leaf_idx = reinterpret_cast<long long*>(take(2 * (size_t)B));
  }
  learner_select_batch(l, 0);
  l->act_tc = take(n_acttc);
  l->q = take(n_lba); l->q_next = take(n_lba); l->target = take(n_lba); l->dq = take(n_lba);
  l->mu = take(n_lba); l->q_pi = take(n_lba); l->dq_pi = take(n_lba); l->dpre_actor = take(n_lba);
  l->td_sq = take((size_t)L * B); l->priority = take(B); l->losses = take(64);
  l->ws_ta = ChainWs::carve(take(ws_ta), l->actor_sh, Tt, B, 1);
  l->ws_tc = ChainWs::carve(take(ws_tc), l->critic_sh, Tt, B, 1);
  l->ws_c1 = ChainWs::carve(take(ws_c1), l->critic_sh, Tc, B, 1);
  l->ws_a1 = ChainWs::carve(take(ws_a1), l->actor_sh, L, B, 2);
  l->ws_c2 = ChainWs::carve(take(ws_c2), l->critic_sh, L, B, 1);
  l->ws_ta.inference_only = true;  // target nets: no BPTT, the scan keeps only what the heads read (learner.py:94-95,106)
  l->ws_tc.inference_only = true;
  for (auto& b : l->slots) {
    b.is_weight = take(B);
    R2D2_TRY(fill_f32(b.is_weight, B, 1.0f, 0));
  }
  l->optim = take(8);
  l->norm_ticket = reinterpret_cast<unsigned int*>(l->optim + 4);   // zeroed with the arena
  l->norm_part = reinterpret_cast<double*>(take(4 * (size_t)kGradNormBlocks));
  if (twin_critic) {
    l->ws_tc_2 = ChainWs::carve(take(ws_tc), l->critic_sh, Tt, B, 1);
    l->ws_c1_2 = ChainWs::carve(take(ws_c1), l->critic_sh, Tc, B, 1);
    l->ws_tc_2.inference_only = true;
    l->q_next2 = take(n_lba); l->q2 = take(n_lba); l->dq2 = take(n_lba);
    l->td_sq2 = take((size_t)L * B);
  }
  R2D2_CUDA_TRY(cudaStreamSynchronize(0));
  learner_select_batch(l, 0);
  {   // R2D2_OVERLAP_INPUTS=0 disables the side and aux streams: the fully serial order (A/B)
    const char* e = getenv("R2D2_OVERLAP_INPUTS");
    l->overlap_inputs = !(e && e[0] == '0');
    if (l->overlap_inputs) {
      int lo = 0, hi = 0;
      R2D2_CUDA_TRY(cudaDeviceGetStreamPriorityRange(&lo, &hi));
      R2D2_CUDA_TRY(cudaStreamCreateWithPriority(&l->side, cudaStreamNonBlocking, lo));   // lowest priority: leftovers only
      // aux at the lowest priority too, a caller's default stream's: a cfg-3 iteration measured 1.2 ms faster than
      // with aux at the highest (DESIGN.md §7)
      R2D2_CUDA_TRY(cudaStreamCreateWithPriority(&l->aux, cudaStreamNonBlocking, lo));
      for (cudaEvent_t* ev : {&l->ev_fork, &l->ev_c1_inputs, &l->ev_a1_inputs, &l->ev_aux_fork, &l->ev_aux_done,
                              &l->ev_q_next_read})
        R2D2_CUDA_TRY(cudaEventCreateWithFlags(ev, cudaEventDisableTiming));
    }
  }
  *out = l;
  return R2D2_OK;
}

int learner_destroy(Learner* l) {
  if (!l) return R2D2_OK;
  if (l->side) { cudaStreamSynchronize(l->side); cudaStreamDestroy(l->side); }
  if (l->aux) { cudaStreamSynchronize(l->aux); cudaStreamDestroy(l->aux); }
  for (cudaEvent_t ev : {l->ev_fork, l->ev_c1_inputs, l->ev_a1_inputs, l->ev_aux_fork, l->ev_aux_done, l->ev_q_next_read})
    if (ev) cudaEventDestroy(ev);
  cudaFree(l->arena);
  cudaFree(l->metrics_part);
  delete l->peer;
  delete l;
  return R2D2_OK;
}

int learner_select_batch(Learner* l, int slot) {
  R2D2_REQUIRE(l && (slot == 0 || slot == 1), "batch slot");
  const Learner::BatchSlot& b = l->slots[slot];
  l->cur_slot = slot;
  l->obs = b.obs; l->act = b.act; l->rew = b.rew; l->term = b.term; l->states = b.states; l->uniforms = b.uniforms;
  l->leaf_idx = b.leaf_idx; l->is_weight = b.is_weight;
  return R2D2_OK;
}

int learner_discard_prefetch(Learner* l, cudaStream_t st) {
  R2D2_REQUIRE(l, "null");
  // whatever the side stream still writes into the online critic's workspace for the dropped batch goes first
  if (l->c1_inputs_slot >= 0 && l->side) R2D2_CUDA_TRY(cudaStreamWaitEvent(st, l->ev_c1_inputs, 0));
  // and whatever the aux stream still reads of the batch in flight (a caller may overwrite either slot next)
  if (l->aux_pending) R2D2_CUDA_TRY(cudaStreamWaitEvent(st, l->ev_aux_done, 0));
  l->c1_inputs_slot = -1;
  l->targets_slot = -1;
  return R2D2_OK;
}

int learner_target_phase(Learner* l, int slot, cudaStream_t st) {
  R2D2_REQUIRE(l && (slot == 0 || slot == 1), "batch slot");
  const r2d2_learner_config& c = l->cfg;
  const int B = c.batch, Bn = c.burn_in, L = c.learning, n = c.n_step, A = c.n_actions, H = c.hidden;
  const int Tt = Bn + n + L, Tc = Bn + L;
  const long long launches0 = launch_count();
  const Learner::BatchSlot& b = l->slots[slot];
  const bool ahead = slot != l->cur_slot;   // batch i+1 while the phases of iteration i are still running on the other slot
  const NetParams Pa_t = NetParams::from_flat(c.target_actor_params, l->actor_sh);
  const NetParams Pc_t = NetParams::from_flat(c.target_critic_params, l->critic_sh);
  const size_t BH = (size_t)B * H;
  const float* st_ta = b.states + 2 * BH;   // states[1] = target_actor (hx, cx)
  const float* st_tc = b.states + 6 * BH;   // states[3] = target_critic

  // target actor over rows [0, Bn+n+L) from its stored state (learner.py:87,94,106); actions for the last L rows
  R2D2_TRY(net_forward_inputs(l->actor_sh, Pa_t, l->ws_ta, b.obs, nullptr, Tt, B, st));
  if (l->overlap_inputs) {
    // fork: input projections that need the batch and weights nothing in this phase changes are issued on a
    // low-priority side stream right where the first persistent scan starts: the scans occupy whole clusters of SMs
    // and the projections take the rest.  Same slot: the online critic chain of this batch (stored actions).  The
    // actor's DPG chain of the iteration in flight: when its weights are final - always when running ahead (the caller
    // completes the previous optimiser step first), else unless the caller defers that step (overlap_actor_inputs).
    bool forked = false;
    auto fork = [&]() -> int {
      if (!forked) {
        R2D2_CUDA_TRY(cudaEventRecord(l->ev_fork, st));
        R2D2_CUDA_TRY(cudaStreamWaitEvent(l->side, l->ev_fork, 0));
        forked = true;
      }
      return R2D2_OK;
    };
    if (!ahead && l->c1_inputs_slot != slot) {
      const NetParams Pc = NetParams::from_flat(c.critic_params, l->critic_sh);
      R2D2_TRY(fork());
      R2D2_TRY(net_forward_inputs(l->critic_sh, Pc, l->ws_c1, b.obs, b.act, Tc, B, l->side));
      R2D2_CUDA_TRY(cudaEventRecord(l->ev_c1_inputs, l->side));
      l->c1_inputs_slot = slot;
    }
    if ((ahead || l->overlap_actor_inputs) && !l->a1_inputs_pending && !l->actor_forward_done) {
      const NetParams Pa = NetParams::from_flat(c.actor_params, l->actor_sh);
      R2D2_TRY(fork());
      R2D2_TRY(net_forward_inputs(l->actor_sh, Pa, l->ws_a1, l->obs + (size_t)Bn * B * c.obs_size, nullptr, L, B, l->side));
      R2D2_CUDA_TRY(cudaEventRecord(l->ev_a1_inputs, l->side));
      l->a1_inputs_pending = true;
    }
  }
  R2D2_TRY(net_forward_scan(l->actor_sh, Pa_t, l->ws_ta, st_ta, st_ta + BH, Tt, B, 1, st));
  // data parallel: this rank's slice sums of whichever gradient block was signalled last - the peers signalled one
  // input projection and one scan ago (peer.cuh); both calls are no-ops without a pending signal
  if (l->peer) {
    R2D2_TRY(peer_reduce(*l->peer, kPeerCritic, st));
    R2D2_TRY(peer_reduce(*l->peer, kPeerActor, st));
  }
  R2D2_CUDA_TRY(cudaMemcpyAsync(l->act_tc, b.act, sizeof(float) * (size_t)(Bn + n) * B * A, cudaMemcpyDeviceToDevice, st));
  float* act_next = l->act_tc + (size_t)(Bn + n) * B * A;
  R2D2_TRY(net_head_forward(l->actor_sh, Pa_t, l->ws_ta, Bn + n, Tt, B, 1, act_next, A, st));
  // TD3 target policy smoothing, in place on the rows the target critics bootstrap from (stored actions stay as they are)
  if (l->target_noise > 0.0f)
    R2D2_TRY(target_smoothing(act_next, act_next, (long long)L * B * A, l->target_noise, l->target_noise_clip,
                              l->noise_seed, l->noise_rank, (unsigned long long)l->critic_iters, st));
  // target critic: stored actions while burning in, target-actor actions afterwards (learner.py:95,106)
  R2D2_TRY(net_forward(l->critic_sh, Pc_t, l->ws_tc, b.obs, l->act_tc, st_tc, st_tc + BH, Tt, B, 1, st));
  if (l->q_next_pending) {   // the twin's TD of the batch in flight, on aux, reads q_next until here
    R2D2_CUDA_TRY(cudaStreamWaitEvent(st, l->ev_q_next_read, 0));
    l->q_next_pending = false;
  }
  R2D2_TRY(net_head_forward(l->critic_sh, Pc_t, l->ws_tc, Bn + n, Tt, B, 1, l->q_next, A, st));
  if (l->twin) {   // target critic 2 from the zero state on the same actions, then q_next = min(q'_1, q'_2)
    const NetParams Pc_t2 = NetParams::from_flat(c.target_critic_params + l->critic_stride(), l->critic_sh);
    R2D2_TRY(net_forward(l->critic_sh, Pc_t2, l->ws_tc_2, b.obs, l->act_tc, nullptr, nullptr, Tt, B, 1, st));
    R2D2_TRY(net_head_forward(l->critic_sh, Pc_t2, l->ws_tc_2, Bn + n, Tt, B, 1, l->q_next2, A, st));
    R2D2_TRY(q_min(l->q_next, l->q_next2, (long long)L * B * A, st));
  }
  l->targets_slot = slot;
  l->launches_target = (int)(launch_count() - launches0);
  return R2D2_OK;
}

int learner_critic_phase(Learner* l, cudaStream_t st) {
  const r2d2_learner_config& c = l->cfg;
  const int B = c.batch, Bn = c.burn_in, L = c.learning, n = c.n_step, A = c.n_actions, H = c.hidden;
  const int Tc = Bn + L;
  const long long launches0 = launch_count();
  const NetParams Pc = NetParams::from_flat(c.critic_params, l->critic_sh);
  const NetParams Gc = NetParams::from_flat(c.critic_grads, l->critic_sh);
  const size_t BH = (size_t)B * H;
  const float* st_c = l->states + 4 * BH;    // states[2] = critic
  const bool concurrent = l->concurrent_chains();
  auto fork_aux = [&]() -> int {
    R2D2_CUDA_TRY(cudaEventRecord(l->ev_aux_fork, st));
    R2D2_CUDA_TRY(cudaStreamWaitEvent(l->aux, l->ev_aux_fork, 0));
    return R2D2_OK;
  };

  // The actor's forward chain reads batch i and the actor weights, which the finish phase of i-1 wrote before this
  // call: on aux it runs beside the target and online critic chains below (the actor phase skips it)
  int actor_launches = 0;
  if (concurrent && !l->actor_forward_done) {
    R2D2_TRY(fork_aux());
    R2D2_TRY(learner_actor_forward(l, l->aux));
    actor_launches = l->launches_actor_forward;
  }
  l->target_phase_standalone = l->targets_slot == l->cur_slot;
  if (!l->target_phase_standalone) R2D2_TRY(learner_target_phase(l, l->cur_slot, st));
  // online critic over rows [0, Bn+L) with stored actions (learner.py:93,105); burn-in stays on the tape (Q4)
  if (l->c1_inputs_slot == l->cur_slot) R2D2_CUDA_TRY(cudaStreamWaitEvent(st, l->ev_c1_inputs, 0));
  else R2D2_TRY(net_forward_inputs(l->critic_sh, Pc, l->ws_c1, l->obs, l->act, Tc, B, st));
  l->c1_inputs_slot = -1;
  R2D2_TRY(net_forward_scan(l->critic_sh, Pc, l->ws_c1, st_c, st_c + BH, Tc, B, 1, st));
  if (l->peer) R2D2_TRY(peer_reduce(*l->peer, kPeerActor, st));   // no target phase in this call: first scan is this one
  R2D2_TRY(net_head_forward(l->critic_sh, Pc, l->ws_c1, Bn, Tc, B, 1, l->q, A, st));
  l->targets_slot = -1;   // q_next is consumed by the TD kernel below

  TdPriorityParams tp;
  tp.q = l->q; tp.q_next = l->q_next; tp.rew = l->rew; tp.term = l->term;
  tp.target = l->target; tp.dq = l->dq; tp.td_sq = l->td_sq; tp.priority = l->priority; tp.loss_sum = l->losses;
  tp.L = L; tp.B = B; tp.A = A; tp.burn_in = Bn; tp.n_step = n;
  tp.gamma_n = (float)std::pow((double)c.gamma, (double)n);
  tp.eta = c.eta;
  tp.is_weight = l->importance_weighting ? l->is_weight : nullptr;
  R2D2_TRY(td_priority(tp, st, TdOptions{l->rescaling, l->rescaling_eps, l->priority_metric}));

  // The priorities exist.  Concurrent chains: the rest of the phase forks onto aux, and the learner stream goes on to
  // the caller's hook and the next batch's target chains; the actor phase joins aux (ev_aux_done) before the critic's
  // Adam.  What the forked work shares with the learner stream until that join, and why each is ordered:
  //   slot i (obs, act, rew, term, is_weight)   read only; the hook writes the other slot
  //   ws_c1 (z1, dG, hs, ...), dq               only the critic phase of i+1 and the side-stream input projection of
  //                                             batch i+1 write them, both issued after the join (the actor phase forks
  //                                             that projection after the critic's Adam)
  //   q, target, priority, losses[0]            written above; the hook only reads the priorities
  //   q_next                                    the twin's TD reads it; the next target phase writes it after waiting
  //                                             for ev_q_next_read
  //   critic_grads, ws_c1_2, q2, dq2, td_sq2, losses[2], metrics partials: aux only until the join
  //   ws_a1, mu (actor forward above)          the actor phase reads them after the join
  //   GEMM operand images, split-K and TD partials: per (device, stream) scratch, aux has its own
  //   act_tc, ws_ta, ws_tc, ws_tc_2, q_next2   the target phase's alone; no forked kernel reads them
  // Data parallel keeps the serial order: a slice-sum kernel spins on SMs that a forked BPTT would need, and the NCCL
  // mode all-reduces the gradients on a stream ordered behind the learner stream only.
  cudaStream_t bs = st;
  if (concurrent) {
    R2D2_TRY(fork_aux());
    bs = l->aux;
  }
  R2D2_CUDA_TRY(cudaMemsetAsync(c.critic_grads, 0, sizeof(float) * l->critic_block(), bs));
  R2D2_TRY(net_backward(l->critic_sh, Pc, &Gc, l->ws_c1, l->obs, l->act, l->dq, Bn, Tc, B, 1, nullptr, nullptr, bs));
  if (l->twin) {
    // critic 2 from the zero state over the same rows with the stored actions, its TD against the same y (q_next is
    // already the minimum; target / priority stay critic 1's), its loss into losses[2], its BPTT into the second half
    const size_t off = l->critic_stride();
    const NetParams Pc2 = NetParams::from_flat(c.critic_params + off, l->critic_sh);
    const NetParams Gc2 = NetParams::from_flat(c.critic_grads + off, l->critic_sh);
    R2D2_TRY(net_forward(l->critic_sh, Pc2, l->ws_c1_2, l->obs, l->act, nullptr, nullptr, Tc, B, 1, bs));
    R2D2_TRY(net_head_forward(l->critic_sh, Pc2, l->ws_c1_2, Bn, Tc, B, 1, l->q2, A, bs));
    TdPriorityParams tp2 = tp;
    tp2.q = l->q2; tp2.target = nullptr; tp2.dq = l->dq2; tp2.td_sq = l->td_sq2; tp2.priority = nullptr;
    tp2.loss_sum = l->losses + 2;
    R2D2_TRY(td_priority(tp2, bs, TdOptions{l->rescaling, l->rescaling_eps, l->priority_metric}));
    if (concurrent) {
      R2D2_CUDA_TRY(cudaEventRecord(l->ev_q_next_read, bs));
      l->q_next_pending = true;
    }
    R2D2_TRY(net_backward(l->critic_sh, Pc2, &Gc2, l->ws_c1_2, l->obs, l->act, l->dq2, Bn, Tc, B, 1, nullptr, nullptr,
                          bs));
  }
  if (l->peer) R2D2_TRY(peer_signal(*l->peer, kPeerCritic, st));
  l->critic_phase_ran = true;
  l->metrics_iter = l->critic_iters;
  if (l->metrics_ring) {
    MetricsCriticParams mp;
    mp.q = l->q; mp.target = l->target; mp.q2 = l->twin ? l->q2 : nullptr; mp.priority = l->priority;
    mp.is_weight = l->importance_weighting ? l->is_weight : nullptr; mp.losses = l->losses;
    mp.n = (long long)L * B * A; mp.B = B; mp.iter = l->metrics_iter; mp.rec = l->metrics_record(l->metrics_iter);
    R2D2_TRY(metrics_critic(mp, l->metrics_part, l->metrics_ticket, bs));
  }
  if (concurrent) {
    R2D2_CUDA_TRY(cudaEventRecord(l->ev_aux_done, l->aux));
    l->aux_pending = true;
  }
  l->critic_iters += 1;
  l->launches_phase[0] = (int)(launch_count() - launches0) - actor_launches;   // the actor phase counts those
  return R2D2_OK;
}

// The actor's forward chain of the DPG update (learner.py:117,120-123 without the critic call): it reads the actor's
// weights and the observations only - NOT the critic - so a data-parallel caller runs it while the all-reduce of the
// critic gradients is in flight (r2d2_learner_actor_forward), before the critic's optimiser step.  A no-op when it already
// ran for this iteration (with concurrent chains the critic phase issues it on aux).
int learner_actor_forward(Learner* l, cudaStream_t st) {
  if (l->actor_forward_done) return R2D2_OK;
  const r2d2_learner_config& c = l->cfg;
  const int B = c.batch, Bn = c.burn_in, L = c.learning, A = c.n_actions, O = c.obs_size;
  const long long launches0 = launch_count();
  const NetParams Pa = NetParams::from_flat(c.actor_params, l->actor_sh);
  const float* obs_l = l->obs + (size_t)Bn * B * O;  // rows [Bn, Bn+L)
  // actor from the zero state, LSTM stepped twice per row (learner.py:117,122-123); mu = output of the 2nd call
  if (l->a1_inputs_pending) {   // issued on the side stream during the critic phase of this iteration
    R2D2_CUDA_TRY(cudaStreamWaitEvent(st, l->ev_a1_inputs, 0));
    l->a1_inputs_pending = false;
  } else {
    R2D2_TRY(net_forward_inputs(l->actor_sh, Pa, l->ws_a1, obs_l, nullptr, L, B, st));
  }
  // data parallel: sum this rank's slice of the critic gradients between the input projection and the scan - the
  // peers signalled one projection ago, the sums are needed one scan later (learner_actor_phase)
  if (l->peer) R2D2_TRY(peer_reduce(*l->peer, kPeerCritic, st));
  R2D2_TRY(net_forward_scan(l->actor_sh, Pa, l->ws_a1, nullptr, nullptr, L, B, 2, st));
  R2D2_TRY(net_head_forward(l->actor_sh, Pa, l->ws_a1, 0, L, B, 2, l->mu, A, st));
  l->actor_forward_done = true;
  l->launches_actor_forward = (int)(launch_count() - launches0);
  return R2D2_OK;
}

// The iteration in flight (l->step + 1 once its finish phase ran) updates the target nets (learner.py:131).
static bool updates_targets(const Learner* l) {
  const int k = l->cfg.target_update_interval;
  return k > 0 && (l->step + 1) % k == 0;
}

// Adam of one net (learner.py:114,128) on the gradient block the optimiser reads - in data-parallel runs the rank sum
// that peer_wait just completed - preceded by the norm kernel when clipping is on, or when metrics are on (the norm
// alone: Adam keeps coef = nullptr, so its instantiation and bits do not change).  On an update iteration with
// target_tau < 1 the net's target is blended in the same pass; target_tau = 1 keeps the finish phase's hard copy.
static int optimiser_step(Learner* l, int block, float* params, float* exp_avg, float* exp_avg_sq, float* target,
                          long long n, float lr, float grad_scale, cudaStream_t st) {
  const float* grads = l->optimiser_grads(block);
  const float* coef = nullptr;
  if (l->grad_clip > 0.0f || l->metrics_ring) {
    R2D2_TRY(grad_norm(grads, n, grad_scale, l->grad_clip, l->norm_part + (size_t)block * kGradNormBlocks,
                       l->norm_ticket + block, l->optim + block, l->optim + 2 + block, st));
    if (l->grad_clip > 0.0f) coef = l->optim + 2 + block;
  }
  const bool polyak = l->target_tau < 1.0f && updates_targets(l);
  return adam_step(params, grads, exp_avg, exp_avg_sq, n, l->step + 1, lr, 0.9f, 0.999f, 1e-8f, grad_scale, st, coef,
                   polyak ? target : nullptr, l->target_tau);
}

int learner_actor_phase(Learner* l, float grad_scale, cudaStream_t st) {
  const r2d2_learner_config& c = l->cfg;
  const int B = c.batch, Bn = c.burn_in, L = c.learning, A = c.n_actions, O = c.obs_size;
  const long long launches0 = launch_count();
  const NetParams Pa = NetParams::from_flat(c.actor_params, l->actor_sh);
  const NetParams Ga = NetParams::from_flat(c.actor_grads, l->actor_sh);
  const NetParams Pc = NetParams::from_flat(c.critic_params, l->critic_sh);
  const long long LBA = (long long)L * B * A;

  if (l->aux_pending) {   // the critic gradients, and the actor's forward chain when the critic phase issued it on aux
    R2D2_CUDA_TRY(cudaStreamWaitEvent(st, l->ev_aux_done, 0));
    l->aux_pending = false;
  }
  int extra = 0;
  if (!l->actor_forward_done) R2D2_TRY(learner_actor_forward(l, st));   // single-GPU order: same kernels, same results
  else extra = l->launches_actor_forward;
  l->actor_forward_done = false;
  const long long launches1 = launch_count();
  (void)launches1;
  if (l->peer) R2D2_TRY(peer_wait(*l->peer, kPeerCritic, st));
  // on an update iteration the critic's target is blended here: nothing later in the iteration changes the critic's
  // weights, and no target chain runs before the iteration ends
  R2D2_TRY(optimiser_step(l, kPeerCritic, c.critic_params, c.critic_exp_avg, c.critic_exp_avg_sq, c.target_critic_params,
                          (long long)l->critic_block(), c.critic_lr, grad_scale, st));   // learner.py:114; twin: both
  {
    // the other slot already holds the next batch (its target chains ran ahead): the input projection of ITS online
    // critic chain needs the weights Adam just wrote and nothing else - side stream, under the scans of this phase
    const int other = 1 - l->cur_slot;
    if (l->overlap_inputs && l->targets_slot == other && l->c1_inputs_slot != other) {
      const Learner::BatchSlot& nb = l->slots[other];
      R2D2_CUDA_TRY(cudaEventRecord(l->ev_fork, st));
      R2D2_CUDA_TRY(cudaStreamWaitEvent(l->side, l->ev_fork, 0));
      R2D2_TRY(net_forward_inputs(l->critic_sh, Pc, l->ws_c1, nb.obs, nb.act, Bn + L, B, l->side));
      R2D2_CUDA_TRY(cudaEventRecord(l->ev_c1_inputs, l->side));
      l->c1_inputs_slot = other;
    }
  }

  const float* obs_l = l->obs + (size_t)Bn * B * O;  // rows [Bn, Bn+L)
  // critic (post-Adam weights, zero state) on the actor's actions; loss = mean(-Q) (learner.py:118,123-124)
  R2D2_TRY(net_forward(l->critic_sh, Pc, l->ws_c2, obs_l, l->mu, nullptr, nullptr, L, B, 1, st));
  R2D2_TRY(net_head_forward(l->critic_sh, Pc, l->ws_c2, 0, L, B, 1, l->q_pi, A, st));
  R2D2_TRY(scaled_sum(l->q_pi, LBA, -1.0f / (float)LBA, l->losses + 1, st));
  if (l->metrics_ring) {   // the critic's norm of this iteration's optimiser step exists by now
    MetricsActorParams mp;
    mp.mu = l->mu; mp.losses = l->losses; mp.critic_norm = l->optim + kPeerCritic; mp.n = LBA;
    mp.rec = l->metrics_record(l->metrics_iter);
    R2D2_TRY(metrics_actor(mp, l->metrics_part, l->metrics_ticket, st));
  }
  R2D2_TRY(fill_f32(l->dq_pi, LBA, -1.0f / (float)LBA, st));
  // dgrad only through the critic (its weight grads are wasted work in the reference); d_pre(actor) = dQ/da * (1-mu^2)
  R2D2_TRY(net_backward(l->critic_sh, Pc, nullptr, l->ws_c2, obs_l, l->mu, l->dq_pi, 0, L, B, 1, l->dpre_actor,
                        l->mu, st));
  R2D2_CUDA_TRY(cudaMemsetAsync(c.actor_grads, 0, sizeof(float) * l->actor_sh.param_count(), st));
  R2D2_TRY(net_backward(l->actor_sh, Pa, &Ga, l->ws_a1, obs_l, nullptr, l->dpre_actor, 0, L, B, 2, nullptr, nullptr, st));
  if (l->peer) R2D2_TRY(peer_signal(*l->peer, kPeerActor, st));
  l->launches_phase[1] = (int)(launch_count() - launches0) + extra;
  return R2D2_OK;
}

int learner_finish_phase(Learner* l, float grad_scale, cudaStream_t st) {
  const r2d2_learner_config& c = l->cfg;
  const long long launches0 = launch_count();
  if (l->peer) R2D2_TRY(peer_wait(*l->peer, kPeerActor, st));   // runs the slice reduction first if no critic phase did
  R2D2_TRY(optimiser_step(l, kPeerActor, c.actor_params, c.actor_exp_avg, c.actor_exp_avg_sq, c.target_actor_params,
                          (long long)l->actor_sh.param_count(), c.actor_lr, grad_scale, st));     // learner.py:128
  // the actor's norm of iteration `step` (which may already be behind the next critic phase): a copy into the ring's
  // side array, no kernel - the host widens it when it reads the record
  if (l->metrics_ring)
    R2D2_CUDA_TRY(cudaMemcpyAsync(l->metrics_actor_norms() + l->step % l->metrics_slots, l->optim + kPeerActor,
                                  sizeof(float), cudaMemcpyDeviceToDevice, st));
  l->step += 1;
  if (l->target_tau == 1.0f && c.target_update_interval > 0 && l->step % c.target_update_interval == 0) {  // :131-132
    R2D2_CUDA_TRY(cudaMemcpyAsync(c.target_actor_params, c.actor_params, sizeof(float) * l->actor_sh.param_count(),
                                  cudaMemcpyDeviceToDevice, st));
    R2D2_CUDA_TRY(cudaMemcpyAsync(c.target_critic_params, c.critic_params, sizeof(float) * l->critic_block(),
                                  cudaMemcpyDeviceToDevice, st));
  }
  l->launches_phase[2] = (int)(launch_count() - launches0);
  return R2D2_OK;
}

int learner_set_metrics(Learner* l, void* ring, int slots) {
  R2D2_REQUIRE(l, "null");
  R2D2_REQUIRE(!ring || slots >= 1, "slots >= 1");
  R2D2_REQUIRE(((uintptr_t)ring & 7) == 0, "the ring holds doubles: 8-byte aligned");
  if (l->critic_phase_ran) {
    set_last_error("metrics are switched on or off before the first critic phase");
    return R2D2_ERR_STATE;
  }
  if (ring && !l->metrics_part) {
    const size_t n = (size_t)kMetricsBlocks * kMetricsPartials;
    R2D2_CUDA_TRY(cudaMalloc(&l->metrics_part, n * sizeof(double) + 64));
    R2D2_CUDA_TRY(cudaMemset(l->metrics_part, 0, n * sizeof(double) + 64));
    R2D2_CUDA_TRY(cudaDeviceSynchronize());   // the ticket is zero before any stream's first metrics kernel
    l->metrics_ticket = reinterpret_cast<unsigned int*>(l->metrics_part + n);
  }
  l->metrics_ring = static_cast<double*>(ring);
  l->metrics_slots = ring ? slots : 0;
  return R2D2_OK;
}

int learner_attach_peers(Learner* l, int rank, int world, void* const* peer_bases) {
  R2D2_REQUIRE(l && peer_bases, "null argument");
  R2D2_REQUIRE(world >= 2 && world <= kPeerMaxWorld && rank >= 0 && rank < world, "peer rank / world");
  R2D2_REQUIRE(!l->peer, "peers already attached");
  PeerExchange* x = new PeerExchange();
  x->rank = rank;
  x->world = world;
  x->lay = peer_layout((long long)l->critic_block(), (long long)l->actor_sh.param_count(), world);
  for (int k = 0; k < world; ++k) {
    if (!peer_bases[k]) { delete x; R2D2_REQUIRE(false, "null peer buffer"); }
    x->ptrs.base[k] = static_cast<char*>(peer_bases[k]);
  }
  l->peer = x;
  l->cfg.critic_grads = x->grads(kPeerCritic);
  l->cfg.actor_grads = x->grads(kPeerActor);
  return R2D2_OK;
}

}  // namespace r2d2

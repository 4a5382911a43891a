// extern "C" surface of libr2d2_b200 (declared in include/r2d2_b200.h).
#include <atomic>
#include <cmath>

#include "common.cuh"
#include "elementwise.cuh"
#include "gemm.cuh"
#include "learner.cuh"
#include "lstm_scan.cuh"
#include "net.cuh"
#include "obs_norm.cuh"
#include "policy.cuh"
#include "replay.cuh"
#include "td3.cuh"

namespace r2d2 {
static thread_local std::string g_last_error;
static std::atomic<long long> g_launches{0};
void set_last_error(const std::string& msg) { g_last_error = msg; }
const char* last_error() { return g_last_error.c_str(); }
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
long long launch_count() { return g_launches.load(std::memory_order_relaxed); }
int num_sms() {
  static std::atomic<int> cache[64];   // 0 = not queried yet
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  int n = cache[dev].load(std::memory_order_relaxed);
  if (n == 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cache[dev].store(n, std::memory_order_relaxed);
  }
  return n;
}
int max_smem_optin() {
  static std::atomic<int> cache[64];   // 0 = not queried yet
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 232448;
  int n = cache[dev].load(std::memory_order_relaxed);
  if (n == 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess || n <= 0) n = 232448;
    cache[dev].store(n, std::memory_order_relaxed);
  }
  return n;
}
}  // namespace r2d2

using namespace r2d2;

static inline cudaStream_t S(r2d2_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }
static inline NetShape shape_of(const r2d2_net_shape* s) {
  return NetShape{s->obs_size, s->n_actions, s->hidden, s->is_critic != 0};
}

extern "C" {

int r2d2_version(void) { return 100; }
long long r2d2_launch_count(void) { return launch_count(); }
const char* r2d2_arch(void) { return "sm_90a"; }
const char* r2d2_last_error(void) { return last_error(); }

int r2d2_device_sm_count(int* out) {
  R2D2_REQUIRE(out, "null");
  int dev = 0;
  R2D2_CUDA_TRY(cudaGetDevice(&dev));
  R2D2_CUDA_TRY(cudaDeviceGetAttribute(out, cudaDevAttrMultiProcessorCount, dev));
  return R2D2_OK;
}

int r2d2_gemm_f32(int layout, int M, int N, int K, const float* A, long long lda, const float* B, long long ldb,
                  const float* A2, long long lda2, const float* B2, long long ldb2, int K2, float* C,
                  long long ldc, const float* bias, const float* Z, long long ldz, int epilogue, int split_k,
                  r2d2_stream_t stream) {
  R2D2_REQUIRE(layout >= 0 && layout <= 2, "layout");
  GemmParams p;
  p.A = A; p.lda = lda; p.B = B; p.ldb = ldb; p.A2 = A2; p.lda2 = lda2; p.B2 = B2; p.ldb2 = ldb2; p.K2 = K2;
  p.C = C; p.ldc = ldc; p.M = M; p.N = N; p.K = K; p.bias = bias; p.Z = Z; p.ldz = ldz; p.epilogue = epilogue;
  p.split_k = split_k < 1 ? 1 : split_k;
  return gemm_f32(p, (GemmLayout)layout, S(stream));
}

size_t r2d2_net_param_count(const r2d2_net_shape* shape) { return shape ? shape_of(shape).param_count() : 0; }

size_t r2d2_net_workspace_floats(const r2d2_net_shape* shape, int T, int B, int repeat) {
  return shape ? ChainWs::floats(shape_of(shape), T, B, repeat) : 0;
}

int r2d2_lstm_net_forward(const r2d2_net_shape* shape, const float* params, const float* obs, const float* act,
                          const float* h0, const float* c0, int T, int B, int repeat, int head_first_row,
                          float* out, float* workspace, r2d2_stream_t stream) {
  R2D2_REQUIRE(shape && params && obs && workspace, "null");
  R2D2_REQUIRE(T > 0 && B > 0 && repeat >= 1, "shape");
  const NetShape s = shape_of(shape);
  const NetParams P = NetParams::from_flat(const_cast<float*>(params), s);
  const ChainWs ws = ChainWs::carve(workspace, s, T, B, repeat);
  R2D2_TRY(net_forward(s, P, ws, obs, act, h0, c0, T, B, repeat, S(stream)));
  if (out) {
    float* ho = ws.head_out + (size_t)head_first_row * B * s.act;
    R2D2_TRY(net_head_forward(s, P, ws, head_first_row, T, B, repeat, ho, s.act, S(stream)));
    R2D2_CUDA_TRY(cudaMemcpyAsync(out, ho, sizeof(float) * (size_t)(T - head_first_row) * B * s.act,
                                  cudaMemcpyDeviceToDevice, S(stream)));
  }
  return R2D2_OK;
}

int r2d2_lstm_net_backward(const r2d2_net_shape* shape, const float* params, const float* obs, const float* act,
                           const float* d_out, int T, int B, int repeat, int head_first_row, float* grads,
                           float* d_act, float* workspace, r2d2_stream_t stream) {
  R2D2_REQUIRE(shape && params && obs && d_out && workspace, "null");
  const NetShape s = shape_of(shape);
  const NetParams P = NetParams::from_flat(const_cast<float*>(params), s);
  const ChainWs ws = ChainWs::carve(workspace, s, T, B, repeat);
  const long long n = (long long)(T - head_first_row) * B * s.act;
  const float* d_pre = d_out;
  if (!s.critic) {  // through the output tanh (models.py:39) using the head outputs kept by the forward call
    R2D2_TRY(mul_dtanh(d_out, ws.head_out + (size_t)head_first_row * B * s.act, ws.d_pre, n, S(stream)));
    d_pre = ws.d_pre;
  }
  NetParams G;
  if (grads) G = NetParams::from_flat(grads, s);
  return net_backward(s, P, grads ? &G : nullptr, ws, obs, act, d_pre, head_first_row, T, B, repeat, d_act, nullptr,
                      S(stream));
}

int r2d2_lstm_scan_forward(const float* gin, const float* whh, const float* h0, const float* c0, float* gates,
                           float* hs, float* cs, float* head_in, int T, int B, int H, int repeat, float* scratch,
                           r2d2_stream_t stream) {
  ScanFwdParams p;
  p.gin = gin; p.whh = whh; p.h0 = h0; p.c0 = c0; p.gates = gates; p.hs = hs; p.cs = cs; p.head_in = head_in;
  p.T = T; p.B = B; p.H = H; p.repeat = repeat; p.scratch = scratch;
  return lstm_scan_forward(p, S(stream));
}

int r2d2_lstm_scan_backward(const float* gates, const float* hs, const float* cs, const float* whh,
                            const float* dh_head, int head_first_step, float* dgates, float* dgin, int T, int B,
                            int H, int repeat, float* scratch, r2d2_stream_t stream) {
  ScanBwdParams p;
  p.gates = gates; p.hs = hs; p.cs = cs; p.whh = whh; p.dh_head = dh_head; p.head_first_step = head_first_step;
  p.dgates = dgates; p.dgin = dgin; p.T = T; p.B = B; p.H = H; p.repeat = repeat; p.scratch = scratch;
  return lstm_scan_backward(p, S(stream));
}

int r2d2_set_gemm_impl(int impl) {
  gemm_set_impl(impl != 0);
  gemm_set_impl_skinny_mma(impl != 2);  // 2 = force the wgmma path even for skinny problems (tests)
  return R2D2_OK;
}
int r2d2_get_gemm_impl(void) { return gemm_get_impl(); }
int r2d2_set_scan_impl(int impl) { lstm_scan_set_impl(impl); return R2D2_OK; }
int r2d2_get_scan_impl(void) { return lstm_scan_get_impl(); }
int r2d2_scan_status(int* status, r2d2_stream_t stream) { return lstm_scan_error_status(status, S(stream)); }

int r2d2_td_priority(const float* q, const float* q_next, const float* rew, const float* term, int L, int B,
                     int A, int burn_in, int n_step, float gamma, float eta, float* target, float* dq,
                     float* td_sq, float* priority, float* critic_loss, r2d2_stream_t stream) {
  TdPriorityParams p;
  p.q = q; p.q_next = q_next; p.rew = rew; p.term = term; p.target = target; p.dq = dq; p.td_sq = td_sq;
  p.priority = priority; p.loss_sum = critic_loss; p.L = L; p.B = B; p.A = A; p.burn_in = burn_in; p.n_step = n_step;
  p.gamma_n = (float)pow((double)gamma, (double)n_step);
  p.eta = eta;
  return td_priority(p, S(stream));
}

int r2d2_td_priority_weighted(const float* q, const float* q_next, const float* rew, const float* term,
                              const float* is_weight, int L, int B, int A, int burn_in, int n_step, float gamma, float eta,
                              float* target, float* dq, float* td_sq, float* priority, float* critic_loss,
                              r2d2_stream_t stream) {
  TdPriorityParams p;
  p.q = q; p.q_next = q_next; p.rew = rew; p.term = term; p.target = target; p.dq = dq; p.td_sq = td_sq;
  p.priority = priority; p.loss_sum = critic_loss; p.L = L; p.B = B; p.A = A; p.burn_in = burn_in; p.n_step = n_step;
  p.gamma_n = (float)pow((double)gamma, (double)n_step);
  p.eta = eta;
  p.is_weight = is_weight;
  return td_priority(p, S(stream));
}

static int td_options_of(const r2d2_td_options* o, TdOptions* out) {
  *out = TdOptions();
  if (o) { out->rescaling = o->rescaling; out->eps = o->eps; out->priority_metric = o->priority_metric; }
  return check_td_options(*out);
}

int r2d2_td_priority_ex(const float* q, const float* q_next, const float* rew, const float* term, const float* is_weight,
                        int L, int B, int A, int burn_in, int n_step, float gamma, float eta, float* target, float* dq,
                        float* td_sq, float* priority, float* critic_loss, const r2d2_td_options* options,
                        r2d2_stream_t stream) {
  TdOptions opt;
  R2D2_TRY(td_options_of(options, &opt));
  TdPriorityParams p;
  p.q = q; p.q_next = q_next; p.rew = rew; p.term = term; p.target = target; p.dq = dq; p.td_sq = td_sq;
  p.priority = priority; p.loss_sum = critic_loss; p.L = L; p.B = B; p.A = A; p.burn_in = burn_in; p.n_step = n_step;
  p.gamma_n = (float)pow((double)gamma, (double)n_step);
  p.eta = eta;
  p.is_weight = is_weight;
  return td_priority(p, S(stream), opt);
}

int r2d2_nstep_rewards(const float* raw, const int* n_rows, int T, int B, int n_step, float gamma, float* out,
                       r2d2_stream_t stream) {
  return nstep_rewards(raw, n_rows, T, B, n_step, gamma, out, S(stream));
}
int r2d2_actor_priorities(const float* q, const float* q_next, const float* rew, const float* term, const int* n_rows,
                          int B, int A, int burn_in, int learning, int n_step, float gamma, float eta, int p_max,
                          float* prio, r2d2_stream_t stream) {
  return actor_priorities(q, q_next, rew, term, n_rows, B, A, burn_in, learning, n_step, gamma, eta, p_max, prio, S(stream));
}
int r2d2_actor_priorities_ex(const float* q, const float* q_next, const float* rew, const float* term, const int* n_rows,
                             int B, int A, int burn_in, int learning, int n_step, float gamma, float eta, int p_max,
                             float* prio, const r2d2_td_options* options, r2d2_stream_t stream) {
  TdOptions opt;
  R2D2_TRY(td_options_of(options, &opt));
  return actor_priorities(q, q_next, rew, term, n_rows, B, A, burn_in, learning, n_step, gamma, eta, p_max, prio,
                          S(stream), opt);
}

size_t r2d2_policy_workspace_floats(const r2d2_net_shape* shape, int N) {
  return shape && N > 0 ? policy_workspace_floats(shape->obs_size, shape->n_actions, shape->hidden, N) : 0;
}

int r2d2_policy_step(const r2d2_net_shape* shape, const float* const params[4], const float* obs,
                     const float* state_in, float* state_out, float* mu, int N, float* workspace,
                     r2d2_stream_t stream) {
  R2D2_REQUIRE(shape, "null");
  return policy_step(shape->obs_size, shape->n_actions, shape->hidden, params, obs, state_in, state_out, mu, N,
                     workspace, S(stream));
}

int r2d2_policy_step_ex(const r2d2_net_shape* shape, const float* const params[4], const float* obs,
                        const float* state_in, float* state_out, float* mu, int N, float* workspace,
                        const float* obs_mean, const float* obs_inv_std, float clip, r2d2_stream_t stream) {
  R2D2_REQUIRE(shape, "null");
  return policy_step(shape->obs_size, shape->n_actions, shape->hidden, params, obs, state_in, state_out, mu, N,
                     workspace, S(stream), obs_mean, obs_inv_std, clip);
}

int r2d2_policy_step_explore(const r2d2_net_shape* shape, const float* const params[4], const float* obs,
                             const float* state_in, float* state_out, float* mu, int N, float* workspace,
                             const float* obs_mean, const float* obs_inv_std, float clip,
                             const r2d2_exploration* exploration, float* action, r2d2_stream_t stream) {
  R2D2_REQUIRE(shape && exploration, "null");
  return policy_step(shape->obs_size, shape->n_actions, shape->hidden, params, obs, state_in, state_out, mu, N,
                     workspace, S(stream), obs_mean, obs_inv_std, clip, exploration, action);
}

int r2d2_obs_norm_merge(double* running, const double* blocks, int W, int O, float* mean_f, float* inv_std_f,
                        r2d2_stream_t stream) {
  return obs_norm_merge(running, blocks, W, O, mean_f, inv_std_f, S(stream));
}
int r2d2_obs_normalize(const float* x, float* y, long long rows, int O, const float* mean_f, const float* inv_std_f,
                       float clip, r2d2_stream_t stream) {
  return obs_normalize(x, y, rows, O, mean_f, inv_std_f, clip, S(stream));
}

int r2d2_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, long long n, int step,
                   float lr, float beta1, float beta2, float eps, float grad_scale, r2d2_stream_t stream) {
  return adam_step(params, grads, exp_avg, exp_avg_sq, n, step, lr, beta1, beta2, eps, grad_scale, S(stream));
}

// ---- replay ----
int r2d2_replay_create(r2d2_replay_t** out, const r2d2_replay_config* cfg) {
  return replay_create(reinterpret_cast<Replay**>(out), cfg, nullptr);
}
int r2d2_replay_create_ex(r2d2_replay_t** out, const r2d2_replay_config* cfg, const r2d2_replay_options* options) {
  return replay_create(reinterpret_cast<Replay**>(out), cfg, options);
}
int r2d2_replay_device_bytes(r2d2_replay_t* r, size_t* out) {
  return replay_device_bytes(reinterpret_cast<Replay*>(r), out);
}
int r2d2_replay_host_bytes(r2d2_replay_t* r, size_t* out) {
  return replay_host_bytes(reinterpret_cast<Replay*>(r), out);
}
int r2d2_replay_destroy(r2d2_replay_t* r) { return replay_destroy(reinterpret_cast<Replay*>(r)); }
int r2d2_replay_set_priority_exponent(r2d2_replay_t* r, float alpha) {
  return replay_set_priority_exponent(reinterpret_cast<Replay*>(r), alpha);
}
int r2d2_replay_add_episode(r2d2_replay_t* r, const float* obs, const float* act, const float* rew,
                            const float* term, const float* states, int n_rows, int n_state_rows,
                            const float* priority, int n_starts, r2d2_stream_t stream) {
  return replay_add_episode(reinterpret_cast<Replay*>(r), obs, act, rew, term, states, n_rows, n_state_rows, priority,
                            n_starts, S(stream));
}
int r2d2_replay_add_episodes(r2d2_replay_t* r, int n_episodes, const int* n_rows, const int* n_starts,
                             const float* obs, const float* act, const float* rew, const float* term,
                             const float* states, const float* leaf_prio, long long* row_start_out,
                             long long* n_evicted_out, long long* sequence_counter_out, r2d2_stream_t stream) {
  return replay_add_episodes(reinterpret_cast<Replay*>(r), n_episodes, n_rows, n_starts, obs, act, rew, term, states,
                             leaf_prio, row_start_out, n_evicted_out, sequence_counter_out, S(stream));
}
int r2d2_replay_add_episodes_ex(r2d2_replay_t* r, int n_episodes, const int* n_rows, const int* n_starts,
                                const float* obs, const float* act, const float* rew, const float* term,
                                const float* states, const float* leaf_prio, long long* row_start_out,
                                long long* n_evicted_out, long long* sequence_counter_out, double* obs_moments,
                                long long* n_nonfinite_out, r2d2_stream_t stream) {
  return replay_add_episodes(reinterpret_cast<Replay*>(r), n_episodes, n_rows, n_starts, obs, act, rew, term, states,
                             leaf_prio, row_start_out, n_evicted_out, sequence_counter_out, S(stream), obs_moments,
                             n_nonfinite_out);
}
int r2d2_replay_set_obs_normalizer(r2d2_replay_t* r, const float* mean_f, const float* inv_std_f, float clip) {
  return replay_set_obs_normalizer(reinterpret_cast<Replay*>(r), mean_f, inv_std_f, clip);
}
int r2d2_replay_sample(r2d2_replay_t* r, const float* u, int batch, long long* leaf_idx, float* obs, float* act,
                       float* rew, float* term, float* states, r2d2_stream_t stream) {
  return replay_sample(reinterpret_cast<Replay*>(r), u, batch, leaf_idx, obs, act, rew, term, states, S(stream));
}
int r2d2_replay_sample_weighted(r2d2_replay_t* r, const float* u, int batch, float beta, long long* leaf_idx,
                                float* is_weight, float* obs, float* act, float* rew, float* term, float* states,
                                r2d2_stream_t stream) {
  return replay_sample_weighted(reinterpret_cast<Replay*>(r), u, batch, beta, leaf_idx, is_weight, obs, act, rew, term,
                                states, S(stream));
}
int r2d2_replay_gather(r2d2_replay_t* r, const long long* leaf_idx, int batch, float* obs, float* act, float* rew,
                       float* term, float* states, r2d2_stream_t stream) {
  return replay_gather(reinterpret_cast<Replay*>(r), leaf_idx, batch, obs, act, rew, term, states, S(stream));
}
int r2d2_replay_update_priorities(r2d2_replay_t* r, const long long* leaf_idx, const float* prio, int batch,
                                  r2d2_stream_t stream) {
  return replay_update_priorities(reinterpret_cast<Replay*>(r), leaf_idx, prio, batch, S(stream));
}
int r2d2_replay_stats(r2d2_replay_t* r, r2d2_replay_stats_t* out, r2d2_stream_t stream) {
  return replay_stats(reinterpret_cast<Replay*>(r), out, S(stream));
}
int r2d2_replay_decode(r2d2_replay_t* r, const long long* leaf_idx_host, int n, long long* episode_index,
                       long long* sequence_index) {
  return replay_decode(reinterpret_cast<Replay*>(r), leaf_idx_host, n, episode_index, sequence_index);
}
int r2d2_replay_tree_level(r2d2_replay_t* r, int level, const float** dev_ptr, long long* n) {
  return replay_tree_level(reinterpret_cast<Replay*>(r), level, dev_ptr, n);
}
int r2d2_replay_export_info(r2d2_replay_t* r, r2d2_replay_snapshot_info* out) {
  return replay_export_info(reinterpret_cast<Replay*>(r), out);
}
int r2d2_replay_export_episodes(r2d2_replay_t* r, long long* row_start, int* n_rows, int* n_starts, long long* serial) {
  return replay_export_episodes(reinterpret_cast<Replay*>(r), row_start, n_rows, n_starts, serial);
}
int r2d2_replay_export_rows(r2d2_replay_t* r, long long first, long long n, float* obs, float* act, float* rew,
                            float* term, void* states, float* leaves, r2d2_stream_t stream) {
  return replay_export_rows(reinterpret_cast<Replay*>(r), first, n, obs, act, rew, term, states, leaves, S(stream));
}
int r2d2_replay_import_begin(r2d2_replay_t* r, const r2d2_replay_snapshot_info* info, const long long* row_start,
                             const int* n_rows, const int* n_starts, const long long* serial, long long* n_dropped_out,
                             r2d2_stream_t stream) {
  return replay_import_begin(reinterpret_cast<Replay*>(r), info, row_start, n_rows, n_starts, serial, n_dropped_out,
                             S(stream));
}
int r2d2_replay_import_rows(r2d2_replay_t* r, long long first, long long n, const float* obs, const float* act,
                            const float* rew, const float* term, const void* states, const float* leaves,
                            r2d2_stream_t stream) {
  return replay_import_rows(reinterpret_cast<Replay*>(r), first, n, obs, act, rew, term, states, leaves, S(stream));
}
int r2d2_replay_import_end(r2d2_replay_t* r, r2d2_stream_t stream) {
  return replay_import_end(reinterpret_cast<Replay*>(r), S(stream));
}

int r2d2_global_layout_for(int rows, int batch, int obs_size, int n_actions, int hidden, int world, r2d2_global_layout* out) {
  R2D2_REQUIRE(out, "null");
  R2D2_REQUIRE(world >= 1 && world <= kGlobalMaxWorld && batch > 0 && rows > 0 && obs_size > 0 && n_actions > 0 &&
               hidden > 0, "global sampling layout arguments");
  const GlobalLayout l = global_layout(rows, batch, obs_size, n_actions, hidden, world);
  out->bytes = l.bytes;
  out->slot_offset[0] = l.slot(0); out->slot_offset[1] = l.slot(1);
  out->off_obs = l.off_obs; out->off_act = l.off_act; out->off_rew = l.off_rew; out->off_term = l.off_term;
  out->off_states = l.off_states; out->off_leaf_idx = l.off_leaf; out->off_shard = l.off_shard;
  out->off_is_weight = l.off_weight; out->off_uniforms = l.off_slot_uniforms;
  return R2D2_OK;
}
int r2d2_replay_attach_group(r2d2_replay_t* r, int rank, int world, int batch, void* const* peer_bases,
                             size_t buffer_bytes) {
  return replay_attach_group(reinterpret_cast<Replay*>(r), rank, world, batch, peer_bases, buffer_bytes);
}
int r2d2_replay_global_write_back(r2d2_replay_t* r, int stage, const long long* leaf_idx, const int* shard,
                                  const float* priority, r2d2_stream_t stream) {
  return replay_global_write_back(reinterpret_cast<Replay*>(r), stage, leaf_idx, shard, priority, S(stream));
}
int r2d2_replay_global_draw(r2d2_replay_t* r, int stage, int slot, int weighted, float beta, r2d2_stream_t stream) {
  return replay_global_draw(reinterpret_cast<Replay*>(r), stage, slot, weighted, beta, S(stream));
}
int r2d2_replay_global_status(r2d2_replay_t* r, int* status, r2d2_stream_t stream) {
  return replay_global_status(reinterpret_cast<Replay*>(r), status, S(stream));
}

// ---- learner ----
int r2d2_learner_create(r2d2_learner_t** out, const r2d2_learner_config* cfg) {
  return learner_create(reinterpret_cast<Learner**>(out), cfg);
}
int r2d2_learner_create_ex(r2d2_learner_t** out, const r2d2_learner_config* cfg, const r2d2_learner_options* options) {
  if (options) R2D2_REQUIRE(options->twin_critic == 0 || options->twin_critic == 1, "twin_critic is 0 or 1");
  return learner_create(reinterpret_cast<Learner**>(out), cfg, options && options->twin_critic == 1);
}
int r2d2_learner_set_target_smoothing(r2d2_learner_t* lh, float sigma, float clip, unsigned int seed, unsigned int rank) {
  R2D2_REQUIRE(lh, "null");
  R2D2_REQUIRE(sigma >= 0.0f && std::isfinite(sigma), "target noise sigma is finite and >= 0 (0 = off)");
  R2D2_REQUIRE(clip > 0.0f && std::isfinite(clip), "target noise clip is finite and > 0");
  Learner* l = reinterpret_cast<Learner*>(lh);
  if (l->targets_slot >= 0) {
    set_last_error("a target phase ran ahead with the old target noise and has not been consumed");
    return R2D2_ERR_STATE;
  }
  l->target_noise = sigma; l->target_noise_clip = clip; l->noise_seed = seed; l->noise_rank = rank;
  return R2D2_OK;
}
int r2d2_learner_twin_buffers(r2d2_learner_t* lh, float** q2, long long* critic2_offset, size_t* twin_bytes) {
  R2D2_REQUIRE(lh && q2 && critic2_offset && twin_bytes, "null");
  Learner* l = reinterpret_cast<Learner*>(lh);
  *q2 = l->q2;
  *critic2_offset = l->twin ? (long long)l->critic_stride() : 0;
  *twin_bytes = l->twin_floats * sizeof(float);
  return R2D2_OK;
}
int r2d2_target_smoothing(const float* mu, float* out, long long n, float sigma, float clip, unsigned int seed,
                          unsigned int rank, unsigned long long iter, r2d2_stream_t stream) {
  R2D2_REQUIRE(std::isfinite(sigma) && std::isfinite(clip), "sigma and clip are finite");
  return target_smoothing(mu, out, n, sigma, clip, seed, rank, iter, S(stream));
}
int r2d2_learner_destroy(r2d2_learner_t* l) { return learner_destroy(reinterpret_cast<Learner*>(l)); }
int r2d2_learner_buffers_get(r2d2_learner_t* lh, r2d2_learner_buffers* o) {
  R2D2_REQUIRE(lh && o, "null");
  Learner* l = reinterpret_cast<Learner*>(lh);
  o->obs = l->obs; o->act = l->act; o->rew = l->rew; o->term = l->term; o->states = l->states;
  o->leaf_idx = l->leaf_idx; o->uniforms = l->uniforms; o->q_value = l->q; o->target_q_value = l->target;
  o->td_sq = l->td_sq; o->priority = l->priority; o->losses = l->losses;
  return R2D2_OK;
}
int r2d2_learner_buffers_get_slot(r2d2_learner_t* lh, int slot, r2d2_learner_buffers* o) {
  R2D2_REQUIRE(lh && o && (slot == 0 || slot == 1), "batch slot");
  Learner* l = reinterpret_cast<Learner*>(lh);
  R2D2_TRY(r2d2_learner_buffers_get(lh, o));
  const Learner::BatchSlot& b = l->slots[slot];
  o->obs = b.obs; o->act = b.act; o->rew = b.rew; o->term = b.term; o->states = b.states;
  o->leaf_idx = b.leaf_idx; o->uniforms = b.uniforms;
  return R2D2_OK;
}
int r2d2_learner_is_weights(r2d2_learner_t* lh, int slot, float** out) {
  R2D2_REQUIRE(lh && out && (slot == 0 || slot == 1), "batch slot");
  *out = reinterpret_cast<Learner*>(lh)->slots[slot].is_weight;
  return R2D2_OK;
}
int r2d2_learner_set_slot_buffers(r2d2_learner_t* lh, int slot, const r2d2_learner_buffers* b, float* is_weight) {
  R2D2_REQUIRE(lh && b && is_weight && (slot == 0 || slot == 1), "batch slot buffers");
  R2D2_REQUIRE(b->obs && b->act && b->rew && b->term && b->states && b->leaf_idx && b->uniforms, "null slot buffer");
  Learner* l = reinterpret_cast<Learner*>(lh);
  if (l->targets_slot >= 0 || l->c1_inputs_slot >= 0) {
    set_last_error("a prefetched batch's chains are pending: move the batch slots before the first step");
    return R2D2_ERR_STATE;
  }
  Learner::BatchSlot& s = l->slots[slot];
  s.obs = b->obs; s.act = b->act; s.rew = b->rew; s.term = b->term; s.states = b->states;
  s.leaf_idx = b->leaf_idx; s.uniforms = b->uniforms; s.is_weight = is_weight;
  return learner_select_batch(l, l->cur_slot);
}
int r2d2_learner_set_importance_weighting(r2d2_learner_t* l, int on) {
  R2D2_REQUIRE(l, "null");
  reinterpret_cast<Learner*>(l)->importance_weighting = on != 0;
  return R2D2_OK;
}
int r2d2_learner_set_target_tau(r2d2_learner_t* l, float tau) {
  R2D2_REQUIRE(l, "null");
  R2D2_REQUIRE(tau > 0.0f && tau <= 1.0f, "target_tau lies in (0, 1]");
  reinterpret_cast<Learner*>(l)->target_tau = tau;
  return R2D2_OK;
}
int r2d2_learner_set_grad_clip(r2d2_learner_t* l, float max_norm) {
  R2D2_REQUIRE(l, "null");
  R2D2_REQUIRE(max_norm >= 0.0f && std::isfinite(max_norm), "max_norm is finite and >= 0 (0 = off)");
  reinterpret_cast<Learner*>(l)->grad_clip = max_norm;
  return R2D2_OK;
}
int r2d2_learner_set_value_rescaling(r2d2_learner_t* l, int mode, float eps) {
  R2D2_REQUIRE(l, "null");
  Learner* e = reinterpret_cast<Learner*>(l);
  TdOptions opt{mode, eps, e->priority_metric};
  R2D2_TRY(check_td_options(opt));
  e->rescaling = mode;
  e->rescaling_eps = mode == kRescaleReference ? 0.0f : eps;
  return R2D2_OK;
}
int r2d2_learner_set_priority_metric(r2d2_learner_t* l, int metric) {
  R2D2_REQUIRE(l, "null");
  Learner* e = reinterpret_cast<Learner*>(l);
  R2D2_TRY(check_td_options(TdOptions{kRescaleReference, 0.0f, metric}));
  e->priority_metric = metric;
  return R2D2_OK;
}
int r2d2_learner_grad_norms(r2d2_learner_t* l, float** out) {
  R2D2_REQUIRE(l && out, "null");
  *out = reinterpret_cast<Learner*>(l)->optim;
  return R2D2_OK;
}
int r2d2_learner_select_batch(r2d2_learner_t* l, int slot) {
  R2D2_REQUIRE(l, "null");
  return learner_select_batch(reinterpret_cast<Learner*>(l), slot);
}
int r2d2_learner_target_phase(r2d2_learner_t* l, int slot, r2d2_stream_t stream) {
  R2D2_REQUIRE(l, "null");
  return learner_target_phase(reinterpret_cast<Learner*>(l), slot, S(stream));
}
int r2d2_learner_discard_prefetch(r2d2_learner_t* l, r2d2_stream_t stream) {
  R2D2_REQUIRE(l, "null");
  return learner_discard_prefetch(reinterpret_cast<Learner*>(l), S(stream));
}
int r2d2_learner_critic_phase(r2d2_learner_t* l, r2d2_stream_t stream) {
  R2D2_REQUIRE(l, "null");
  return learner_critic_phase(reinterpret_cast<Learner*>(l), S(stream));
}
int r2d2_learner_actor_forward(r2d2_learner_t* l, r2d2_stream_t stream) {
  R2D2_REQUIRE(l, "null");
  return learner_actor_forward(reinterpret_cast<Learner*>(l), S(stream));
}
int r2d2_learner_actor_phase(r2d2_learner_t* l, float grad_scale, r2d2_stream_t stream) {
  R2D2_REQUIRE(l, "null");
  return learner_actor_phase(reinterpret_cast<Learner*>(l), grad_scale, S(stream));
}
int r2d2_learner_finish_phase(r2d2_learner_t* l, float grad_scale, r2d2_stream_t stream) {
  R2D2_REQUIRE(l, "null");
  return learner_finish_phase(reinterpret_cast<Learner*>(l), grad_scale, S(stream));
}
int r2d2_learner_step_count(r2d2_learner_t* l) { return l ? reinterpret_cast<Learner*>(l)->step : -1; }
int r2d2_learner_set_overlap_actor_inputs(r2d2_learner_t* l, int on) {
  R2D2_REQUIRE(l, "null");
  reinterpret_cast<Learner*>(l)->overlap_actor_inputs = on != 0;
  return R2D2_OK;
}
int r2d2_peer_layout_for(long long n_critic, long long n_actor, int world, r2d2_peer_layout* out) {
  R2D2_REQUIRE(out && n_critic > 0 && n_actor > 0 && world >= 2 && world <= kPeerMaxWorld, "peer layout arguments");
  const PeerLayout pl = peer_layout(n_critic, n_actor, world);
  out->bytes = pl.bytes;
  out->off_critic_grads = pl.off_grads[kPeerCritic];
  out->off_actor_grads = pl.off_grads[kPeerActor];
  out->off_critic_sums = pl.off_sums[kPeerCritic];
  out->off_actor_sums = pl.off_sums[kPeerActor];
  return R2D2_OK;
}
int r2d2_learner_peer_layout(r2d2_learner_t* lh, int world, r2d2_peer_layout* out) {
  R2D2_REQUIRE(lh && out && world >= 2 && world <= kPeerMaxWorld, "peer layout arguments");
  Learner* l = reinterpret_cast<Learner*>(lh);
  const PeerLayout pl = peer_layout((long long)l->critic_block(), (long long)l->actor_sh.param_count(), world);
  out->bytes = pl.bytes;
  out->off_critic_grads = pl.off_grads[kPeerCritic];
  out->off_actor_grads = pl.off_grads[kPeerActor];
  out->off_critic_sums = pl.off_sums[kPeerCritic];
  out->off_actor_sums = pl.off_sums[kPeerActor];
  return R2D2_OK;
}
int r2d2_learner_attach_peers(r2d2_learner_t* l, int rank, int world, void* const* peer_bases) {
  return learner_attach_peers(reinterpret_cast<Learner*>(l), rank, world, peer_bases);
}
int r2d2_learner_peer_status(r2d2_learner_t* lh, int* status, r2d2_stream_t stream) {
  R2D2_REQUIRE(lh && status, "null");
  Learner* l = reinterpret_cast<Learner*>(lh);
  R2D2_REQUIRE(l->peer, "no peers attached");
  return peer_status(*l->peer, status, static_cast<cudaStream_t>(stream));
}
int r2d2_learner_peer_counters(r2d2_learner_t* lh, unsigned long long* out6, int reset, r2d2_stream_t stream) {
  R2D2_REQUIRE(lh && out6, "null");
  Learner* l = reinterpret_cast<Learner*>(lh);
  R2D2_REQUIRE(l->peer, "no peers attached");
  return peer_counters(*l->peer, out6, reset, static_cast<cudaStream_t>(stream));
}
int r2d2_learner_set_step_count(r2d2_learner_t* l, int step) {
  R2D2_REQUIRE(l && step >= 0, "step");
  reinterpret_cast<Learner*>(l)->step = step;
  reinterpret_cast<Learner*>(l)->critic_iters = step;   // the target noise's iteration index resumes with it
  return R2D2_OK;
}
size_t r2d2_metrics_ring_bytes(int slots) {
  return slots >= 1 ? (size_t)slots * (kMetricsFields * sizeof(double) + sizeof(float)) : 0;
}
int r2d2_metrics_field_count(void) { return kMetricsFields; }
const char* r2d2_metrics_field_name(int i) { return metrics_field_name(i); }
int r2d2_learner_set_metrics(r2d2_learner_t* l, void* ring, int slots) {
  return learner_set_metrics(reinterpret_cast<Learner*>(l), ring, slots);
}
int r2d2_learner_launches_per_iteration(r2d2_learner_t* lh) {
  if (!lh) return -1;
  Learner* l = reinterpret_cast<Learner*>(lh);
  return l->launches_phase[0] + l->launches_phase[1] + l->launches_phase[2] +
         (l->target_phase_standalone ? l->launches_target : 0);
}

}  // extern "C"

/* libr2d2_b200 - C ABI of the GPU-native (H100, sm_90a) learner hot path of pytorch-r2d2-DPG.
 *
 * The reference (pure Python) has no FFI; its boundary for this path is the module surface
 * learner.py / replay_memory.py / models.py / utils.py.  Each entry point below replaces the
 * reference function(s) cited next to it; the host-side mirror in pytorch-r2d2-dpg_b200/*.py binds
 * them with ctypes (see INTEGRATION.md).
 *
 * Conventions
 *   - every function returns 0 on success, <0 on error; r2d2_last_error() (thread-local) has the text;
 *   - tensors are caller-owned device memory (fp32, contiguous, time-major [T,B,*] as produced by
 *     replay_memory.py:123-136), passed as raw pointers + explicit sizes; no torch types here;
 *   - the library owns only opaque handles (replay shard + sum tree, learner workspaces);
 *   - every launch goes to the cudaStream_t given (passed as void*); nothing synchronises the host
 *     unless stated; one host thread per handle.
 *   - parameter blocks are FLAT fp32 buffers in the reference's state_dict order
 *     (l1.weight[H,I], l1.bias[H], l2.weight_ih[4H,H], l2.weight_hh[4H,H], l2.bias_ih[4H],
 *      l2.bias_hh[4H], l3.weight[A,H], l3.bias[A]; models.py:17-19,59-61), I = O (actor) or O+A (critic).
 */
#ifndef R2D2_B200_H_
#define R2D2_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define R2D2_OK 0
#define R2D2_ERR_CUDA (-1)
#define R2D2_ERR_ARG (-2)
#define R2D2_ERR_UNSUPPORTED (-3)
#define R2D2_ERR_STATE (-4)

typedef void* r2d2_stream_t; /* cudaStream_t */

int r2d2_version(void);                /* 100 * major + minor */
/* kernels this process has launched through the library so far (launch budgets of the entry points) */
long long r2d2_launch_count(void);
const char* r2d2_arch(void);           /* "sm_90a" */
const char* r2d2_last_error(void);
int r2d2_device_sm_count(int* out);

/* ------------------------------------------------------------------------------------------------
 * Dense building block (x*W^T, dgrad, wgrad of models.py:33,37-39,76,80-82): fp32 in/out, bf16x3
 * tensor-core MMAs.  layout: 0 = NT (A[M,K] * B[N,K]^T), 1 = NN (A[M,K] * B[K,N]), 2 = TN (A[K,M]^T * B[K,N]).
 * epilogue: 0 none, 1 tanh(acc+bias), 2 (acc+bias)*(1-Z^2), 3 acc+bias+Z.  split_k > 1 adds into C.
 * ---------------------------------------------------------------------------------------------- */
int r2d2_gemm_f32(int layout, int M, int N, int K, const float* A, long long lda, const float* B, long long ldb,
                  const float* A2, long long lda2, const float* B2, long long ldb2, int K2, float* C,
                  long long ldc, const float* bias, const float* Z, long long ldz, int epilogue, int split_k,
                  r2d2_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Recurrent net chains: replace the per-timestep python loops over ActorNet/CriticNet.__call__
 * (models.py:32-40,74-83) at learner.py:92-95,102-106,120-123.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  int obs_size;   /* O */
  int n_actions;  /* A */
  int hidden;     /* H (128 in the reference, models.py:17-19) */
  int is_critic;  /* 0: ActorNet, 1: CriticNet (input = cat(obs, action), head without tanh, A outputs) */
} r2d2_net_shape;

size_t r2d2_net_param_count(const r2d2_net_shape* shape);
/* floats of workspace needed by one chain of T input rows, `repeat` cell steps per row, batch B */
size_t r2d2_net_workspace_floats(const r2d2_net_shape* shape, int T, int B, int repeat);

/* Forward over T rows (S = T*repeat cell steps).  obs [T,B,O]; act [T,B,A] (critic only, else NULL);
 * h0/c0 [B,H] or NULL for the zero state (models.py:34-36).  Head outputs are produced for input rows
 * [head_first_row, T) (after the last of the `repeat` steps of each row) into out [(T-head_first_row),B,A].
 * workspace keeps the activations for r2d2_lstm_net_backward. */
int r2d2_lstm_net_forward(const r2d2_net_shape* shape, const float* params, const float* obs, const float* act,
                          const float* h0, const float* c0, int T, int B, int repeat, int head_first_row,
                          float* out, float* workspace, r2d2_stream_t stream);

/* BPTT through the chain saved in `workspace`.  d_out [(T-head_first_row),B,A] = dLoss/d(head output).
 * grads: flat buffer like params, ACCUMULATED into (zero it first); NULL -> data gradient only.
 * d_act [T,B,A]: dLoss/d(action input) (critic only, optional).  The workspace is consumed. */
int r2d2_lstm_net_backward(const r2d2_net_shape* shape, const float* params, const float* obs, const float* act,
                           const float* d_out, int T, int B, int repeat, int head_first_row, float* grads,
                           float* d_act, float* workspace, r2d2_stream_t stream);

/* The serial scan alone (the persistent-RNN kernel; bench.py times it for the roofline line):
 * gin [T,B,4H] pre-activation input projection, whh [4H,H], h0/c0 [B,H] or NULL; outputs gates [T*repeat,B,4H]
 * (may alias gin when repeat == 1), hs/cs [T*repeat+1,B,H], head_in [T,B,H] or NULL.  scratch: [B,4H] floats
 * (used by the per-step path; NULL is accepted when the cluster kernels cover H and are selected). */
int r2d2_lstm_scan_forward(const float* gin, const float* whh, const float* h0, const float* c0, float* gates,
                           float* hs, float* cs, float* head_in, int T, int B, int H, int repeat, float* scratch,
                           r2d2_stream_t stream);
/* BPTT twin: dgates [S,B,4H] (may alias gates), dgin [T,B,4H] (only when repeat > 1), dh_head [*,B,H] or NULL
 * consumed from step head_first_step on.  scratch: [2,B,H] (NULL as for the forward scan). */
int r2d2_lstm_scan_backward(const float* gates, const float* hs, const float* cs, const float* whh,
                            const float* dh_head, int head_first_step, float* dgates, float* dgin, int T, int B,
                            int H, int repeat, float* scratch, r2d2_stream_t stream);

/* GEMM implementation switch for A/B checks: 1 = wgmma with skinny problems (K<64, N<32 or M<32) on the fp32
 * streaming / single-launch mma.sync kernels (default), 2 = wgmma for every shape, 0 = mma.sync kernel only */
int r2d2_set_gemm_impl(int impl);
int r2d2_get_gemm_impl(void);
/* scan implementation switch for A/B checks: 1 = persistent cluster kernels where they cover H (default),
 * 0 = per-step path (one GEMM + one cell kernel per step) for every H */
int r2d2_set_scan_impl(int impl);
int r2d2_get_scan_impl(void);
/* *status != 0 if a scan kernel reported a protocol error; synchronises the stream */
int r2d2_scan_status(int* status, r2d2_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Fused n-step target + value rescaling + TD loss gradient + sequence priority
 * (learner.py:107-111,135-138; utils.py:17-21).  q, q_next [L,B,A]; rew, term [T',B].
 * Any output pointer may be NULL.
 * ---------------------------------------------------------------------------------------------- */
int r2d2_td_priority(const float* q, const float* q_next, const float* rew, const float* term, int L, int B,
                     int A, int burn_in, int n_step, float gamma, float eta, float* target, float* dq,
                     float* td_sq, float* priority, float* critic_loss, r2d2_stream_t stream);
/* The same with importance-sampling weights is_weight [B] (DEVICE, from r2d2_replay_sample_weighted; NULL = all 1):
 * dq = w_b * 2 (q - y) / (L*B*A) and critic_loss = sum w_b td_sq / (L*B).  td_sq and priority stay unweighted (a
 * sequence's priority does not depend on how it was drawn).  w = 1 gives the bits of r2d2_td_priority. */
int r2d2_td_priority_weighted(const float* q, const float* q_next, const float* rew, const float* term,
                              const float* is_weight, int L, int B, int A, int burn_in, int n_step, float gamma, float eta,
                              float* target, float* dq, float* td_sq, float* priority, float* critic_loss,
                              r2d2_stream_t stream);

/* n-step target and priority options (published R2D2; neither is in the reference):
 *   rescaling  R2D2_RESCALE_REFERENCE (default): y = h0(R + gamma^n (1-d) Q'), h0(x) = sign(x)(sqrt(|x|+1) - 1) - no eps x
 *              term and no inverse on the bootstrap (utils.py:20-21, learner.py:107-108);
 *              R2D2_RESCALE_INVERTIBLE: y = h_eps(R + gamma^n (1-d) h_eps^-1(Q')), h_eps(x) = h0(x) + eps x, in forms that
 *              keep fp32 accurate near 0: h_eps(x) = sign(x) |x| / (sqrt(|x|+1) + 1) + eps x and
 *              h_eps^-1(x) = sign(x) v (v+2), v = 2|x| / ((1+2eps) + sqrt((1+2eps)^2 + 4 eps |x|)).
 *              The loss stays the MSE against y; target, dq and td_sq keep their meaning.
 *   eps        h_eps's eps in [0, 1] (R2D2: 1e-3); ignored by the reference rescaling.
 *   priority_metric  R2D2_PRIORITY_SQUARED (default): eta max + (1-eta) mean of td_sq (utils.py:17-18);
 *              R2D2_PRIORITY_ABS: of m = sqrt(td_sq), the RMS over the A actions = |delta| at A = 1.  td_sq and the loss
 *              do not change.
 * NULL options = the defaults, the kernels and bits of the entries without _ex.  An unknown mode or metric, or (invertible)
 * an eps that is NaN, inf, negative or > 1, is R2D2_ERR_ARG. */
#define R2D2_RESCALE_REFERENCE 0
#define R2D2_RESCALE_INVERTIBLE 1
#define R2D2_PRIORITY_SQUARED 0
#define R2D2_PRIORITY_ABS 1
typedef struct {
  int rescaling;
  float eps;
  int priority_metric;
} r2d2_td_options;
/* r2d2_td_priority_weighted (is_weight may be NULL) with options */
int r2d2_td_priority_ex(const float* q, const float* q_next, const float* rew, const float* term, const float* is_weight,
                        int L, int B, int A, int burn_in, int n_step, float gamma, float eta, float* target, float* dq,
                        float* td_sq, float* priority, float* critic_loss, const r2d2_td_options* options,
                        r2d2_stream_t stream);

/* Actor-side rows of the path (SURVEY 8f N2), batched over finished episodes (one episode per batch column, time-major,
 * zero padded): n-step discounted reward pre-sum (actor.py:74-76; rows i < n_rows[b] - n_step, later rows copied) and
 * the initial sequence priorities (actor.py:78-107): priority k = eta*max + (1-eta)*mean over j = k+burn_in+1 ..
 * k+burn_in+learning of (mean_A(q[j] - h(R[j] + gamma^n (1-term[j+n-1]) q_next[j+n])))^2 - the reference's deque is one
 * step ahead of the learner's window and squares the MEAN difference; both are kept.  prio [B, p_max], zero where
 * k >= n_rows[b] - n_step - burn_in - learning.  q, q_next come from r2d2_lstm_net_forward on the zero state. */
int r2d2_nstep_rewards(const float* raw, const int* n_rows, int T, int B, int n_step, float gamma, float* out,
                       r2d2_stream_t stream);
int r2d2_actor_priorities(const float* q, const float* q_next, const float* rew, const float* term, const int* n_rows,
                          int B, int A, int burn_in, int learning, int n_step, float gamma, float eta, int p_max,
                          float* prio, r2d2_stream_t stream);
/* r2d2_actor_priorities with options (r2d2_td_options): the invertible target, and under R2D2_PRIORITY_ABS |td| in place
 * of td^2 - td still the MEAN difference over actions, where the learner's abs metric takes the RMS; the actor and the
 * learner differ here as they do in the squared metric. */
int r2d2_actor_priorities_ex(const float* q, const float* q_next, const float* rew, const float* term, const int* n_rows,
                             int B, int A, int burn_in, int learning, int n_step, float gamma, float eta, int p_max,
                             float* prio, const r2d2_td_options* options, r2d2_stream_t stream);

/* Actor side, per env step: the four nets of N actor lanes stepped once (Actor.run, actor.py:149-154).
 * shape: O, A, H (is_critic ignored).  params: flat blocks of actor, target_actor, critic, target_critic (the critics'
 * I = O + A).  obs [N,O]; state_in, state_out [4,2,N,H] in that net order, (hx, cx) - the replay's state layout;
 * they must not alias.  mu [N,A] = tanh(l3(tanh(h'))) of the actor, before any exploration noise.  The critics are fed
 * cat(obs, mu) and the target critic cat(obs, mu_t); the critics' heads are not computed (the reference discards them).
 * fp32 FMA on the flat weights; lane n's outputs are bitwise independent of N and of the other lanes.  Five kernel
 * launches on `stream`, no host synchronisation.  Supported: 1 <= N <= 256, H a multiple of 32 up to 512, 1 <= A <= 64;
 * other shapes return R2D2_ERR_UNSUPPORTED.  workspace: r2d2_policy_workspace_floats(shape, N) floats. */
size_t r2d2_policy_workspace_floats(const r2d2_net_shape* shape, int N);
int r2d2_policy_step(const r2d2_net_shape* shape, const float* const params[4], const float* obs,
                     const float* state_in, float* state_out, float* mu, int N, float* workspace,
                     r2d2_stream_t stream);

/* r2d2_policy_step with an observation normaliser: obs_mean, obs_inv_std DEVICE [O] (both or neither; NULL is
 * r2d2_policy_step), clip finite and > 0.  Phase 1 reads x_hat = clamp(fl(fl(x - mean) * inv_std), -clip, clip) (NaN
 * passes through) in place of every obs value as it stages the obs rows - the bits r2d2_obs_normalize writes - so the
 * step equals r2d2_policy_step on pre-normalised obs bit for bit; lane n's outputs stay independent of N.  Same five
 * launches, the first one a separate kernel. */
int r2d2_policy_step_ex(const r2d2_net_shape* shape, const float* const params[4], const float* obs,
                        const float* state_in, float* state_out, float* mu, int N, float* workspace,
                        const float* obs_mean, const float* obs_inv_std, float clip, r2d2_stream_t stream);

/* Actor exploration noise drawn in the step (off unless a caller asks for it; the reference adds N(0, 0.3) on the host).
 * For lane n and action a, z comes from the generator of r2d2_target_smoothing with key = (seed, actor_id[n]) and
 * counter = (a >> 2, (uint32) step, step >> 32, 1) - words (x0, x1) serve a % 4 in {0, 1}, (x2, x3) serve {2, 3}, the
 * same Box-Muller - so c3 = 1 keeps these streams apart from target smoothing's (c3 = 0), and lane n's noise depends
 * on its actor id and the step only, never on N or on the lane's position.  In fp32, in this order:
 *   R2D2_EXPLORATION_GAUSSIAN: noise = fl(sigma[n] z)
 *   R2D2_EXPLORATION_OU:       x' = fl(fl(one_minus_theta x) + fl(sigma[n] z)), written back to x = ou_state[n, a];
 *                              noise = x'
 *   action[n, a] = min(max(fl(mu[n, a] + noise), -1), 1)
 * mu stays the noise-free actor output, and the critics read it. */
#define R2D2_EXPLORATION_GAUSSIAN 0
#define R2D2_EXPLORATION_OU 1
typedef struct {
  int kind;                    /* R2D2_EXPLORATION_GAUSSIAN or R2D2_EXPLORATION_OU; anything else is R2D2_ERR_ARG */
  unsigned int seed;           /* first key word of every lane's stream */
  unsigned long long step;     /* the actors' 0-based env-step count: the counter's words 1 and 2 */
  float one_minus_theta;       /* OU: fl32(1 - theta), theta in (0, 1] so in [0, 1); ignored for GAUSSIAN */
  const unsigned int* actor_id;  /* DEVICE [N]: the second key word of lane n */
  const float* sigma;          /* DEVICE [N]: lane n's noise scale, finite and >= 0 */
  float* ou_state;             /* DEVICE [N, A], read and written: OU's x (zero it at a lane's episode start); NULL for
                                  GAUSSIAN */
} r2d2_exploration;
/* r2d2_policy_step_ex (obs_mean NULL: the raw-obs path) that also writes action [N, A] (DEVICE; must not overlap mu)
 * as defined above, from the actor head's registers; mu, the target actor's mu_t, the critics' inputs and every state
 * are bitwise those of r2d2_policy_step_ex.  Same five launches: the head phase is a separate kernel.  Before any
 * launch the call copies sigma [N] to the host and synchronises `stream` to check it; a sigma that is NaN, inf or
 * negative, one_minus_theta outside [0, 1) under OU, a NULL pointer where one is needed, a non-NULL ou_state under
 * GAUSSIAN, an unknown kind or overlapping action and mu is R2D2_ERR_ARG; unsupported shapes are R2D2_ERR_UNSUPPORTED
 * as for r2d2_policy_step.  Nothing is launched on an error. */
int r2d2_policy_step_explore(const r2d2_net_shape* shape, const float* const params[4], const float* obs,
                             const float* state_in, float* state_out, float* mu, int N, float* workspace,
                             const float* obs_mean, const float* obs_inv_std, float clip,
                             const r2d2_exploration* exploration, float* action, r2d2_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Observation normalisation (off unless a caller attaches it).  Statistics are moment blocks of [1 + 2 O] doubles:
 * count, mean [O], M2 [O] (the sum of squared deviations from the mean).  The fp32 pair every transform reads is
 * mean_f = (float) mean, inv_std_f = (float)(1 / sqrt(M2 / n + 1e-8)), each rounded once from double, and the transform
 * is x_hat = clamp(fl(fl(x - mean_f) * inv_std_f), -clip, clip) with NaN passing through (torch.clamp's behaviour).
 * ---------------------------------------------------------------------------------------------- */
/* Merge W blocks (DEVICE [W, 1 + 2 O]) into `running` (DEVICE [1 + 2 O]) in index order with Chan's parallel formula
 * (n = na + nb, d = mb - ma, mean = ma + d nb / n, M2 = M2a + M2b + d^2 na nb / n; an empty side takes the other's values
 * unchanged), then rewrite DEVICE mean_f, inv_std_f [O] from it; with n = 0 they become 0 and 1.  mean_f and inv_std_f
 * may both be NULL (merge only).  One single-CTA launch, deterministic. */
int r2d2_obs_norm_merge(double* running, const double* blocks, int W, int O, float* mean_f, float* inv_std_f,
                        r2d2_stream_t stream);
/* y [rows, O] = x_hat of x [rows, O] (DEVICE; y may be x).  One grid-stride launch. */
int r2d2_obs_normalize(const float* x, float* y, long long rows, int O, const float* mean_f, const float* inv_std_f,
                       float clip, r2d2_stream_t stream);

/* torch.optim.Adam defaults (learner.py:50-53,114,128) on a flat buffer; grad is multiplied by grad_scale first. */
int r2d2_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, long long n, int step,
                   float lr, float beta1, float beta2, float eps, float grad_scale, r2d2_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * GPU-resident prioritized sequence replay (replaces LearnerReplayMemory, replay_memory.py:67-175).
 * Rows of all episodes live in HBM (SoA); one sum-tree leaf per row (priority 0 for rows that are
 * not valid sequence starts); 32-ary tree of fp32 partial sums.  P(start) is proportional to its
 * priority, which is what the reference's two-level draw (replay_memory.py:95-114) samples.
 * ---------------------------------------------------------------------------------------------- */
typedef struct r2d2_replay r2d2_replay_t;

typedef struct {
  int obs_size, n_actions, hidden;
  int burn_in, learning, n_step;   /* window rows T' = burn_in + learning + n_step (replay_memory.py:116) */
  long long capacity_rows;         /* physical rows in HBM (ring) */
  long long max_sequences;         /* eviction threshold on the sequence counter (replay_memory.py:148) */
} r2d2_replay_config;

int r2d2_replay_create(r2d2_replay_t** out, const r2d2_replay_config* cfg);

/* Storage precision of the recurrent states [4,2,H] of every row (obs, act, rew, term and the tree stay fp32).
 * R2D2_STATE_F16 halves the bytes of the states, which are most of a row (91 % at O 376, A 17, H 512).  The states are
 * rounded once at ingest (IEEE round-to-nearest-even) and widened exactly by the gather, so the batch holds exactly the
 * fp16-rounded inputs.  The bound that makes fp16 safe: h = o tanh(c) gives |h| < 1, and c_t = f c_{t-1} + i g with
 * f, i in (0, 1), |g| < 1 and c_0 = 0 gives |c_t| < t, so only an episode longer than 65,504 steps could overflow;
 * the relative rounding error is at most 2^-12 (bf16's 2^-9 would exceed a 1e-3 parity bar on its own).  States from
 * foreign actors can hold anything, so ingest in this mode checks: a finite value of magnitude >= 65520 (which would
 * round to +-inf) refuses the whole add_episode(s) call with R2D2_ERR_ARG, naming the count, before any episode is
 * placed, evicted or committed - the shard, its tree and its counters stay as they were.  NaN and +-inf pass through,
 * as in fp32 storage.  Ingest in this mode copies the states into a grow-only device staging block and adds two
 * kernels and one stream synchronisation per call; the gather is still one launch. */
#define R2D2_STATE_F32 0
#define R2D2_STATE_F16 1
/* Where the recurrent states [cap,4,2,H] live.  R2D2_STATE_MEMORY_HOST puts them in mapped, page-locked host memory
 * (cudaHostAlloc, zeroed at creation; no fallback to HBM if it fails) while obs, act, rew, term and the whole sum tree
 * stay in HBM.  The learner reads the states only at a window's first row, one [8,H] block per drawn sequence (7.7 % of
 * a cfg-3 batch's gather bytes), so the gather reads them over the host link and the HBM a row needs drops to
 * 4 (O + A + 2) + 5 bytes.  The batch is bit-identical to the device tier's.  Every write to the host rows is ordered
 * on the caller's stream: ingest and restore stage the states in a grow-only device block (fp32 storage adds one
 * device-to-host copy per contiguous ring run, fp16 storage writes the rounded states straight from its conversion
 * kernel), so a write never overtakes a gather issued earlier on the same stream. */
#define R2D2_STATE_MEMORY_DEVICE 0
#define R2D2_STATE_MEMORY_HOST 1
typedef struct {
  int state_storage;   /* R2D2_STATE_F32 (default) or R2D2_STATE_F16; anything else is R2D2_ERR_ARG */
  int state_memory;    /* R2D2_STATE_MEMORY_DEVICE (default) or R2D2_STATE_MEMORY_HOST; anything else is R2D2_ERR_ARG */
} r2d2_replay_options;
/* options NULL (or a zeroed struct) = r2d2_replay_create */
int r2d2_replay_create_ex(r2d2_replay_t** out, const r2d2_replay_config* cfg, const r2d2_replay_options* options);
/* bytes of device memory the shard holds (rows, tree, and the staging block once an ingest or restore has used it);
 * under R2D2_STATE_MEMORY_HOST the states are not device memory and are not counted here */
int r2d2_replay_device_bytes(r2d2_replay_t* r, size_t* out);
/* bytes of pinned host memory the shard holds: cap * 8 H * sizeof(state) under R2D2_STATE_MEMORY_HOST, else 0 */
int r2d2_replay_host_bytes(r2d2_replay_t* r, size_t* out);
int r2d2_replay_destroy(r2d2_replay_t* r);
/* Priority exponent alpha in [0, 1] (prioritized replay; default 1 = the raw priority): every leaf the shard writes -
 * ingest and r2d2_replay_update_priorities - holds p > 0 ? p^alpha : 0, so P(start) = p^alpha / sum p^alpha and rows
 * that start no sequence stay undrawable even at alpha = 0 (uniform over valid starts).  Callers keep passing raw
 * priorities.  Only while the shard holds no episode (else R2D2_ERR_STATE); alpha outside [0, 1] is R2D2_ERR_ARG. */
int r2d2_replay_set_priority_exponent(r2d2_replay_t* r, float alpha);

/* Append one episode (replay_memory.py:141-152).  HOST pointers: obs [n_rows,O], act [n_rows,A], rew [n_rows],
 * term [n_rows] (n_rows includes the n_step pad rows, actor.py:173), states [n_state_rows,4,2,H]
 * (actor, target_actor, critic, target_critic) x (hx,cx), priority [n_starts].  Oldest episodes are
 * evicted FIFO when the ring overflows, and after the append while the sequence counter exceeds max_sequences - the
 * rules of a one-episode r2d2_replay_add_episodes, which may evict the new episode too.  Synchronises the stream. */
int r2d2_replay_add_episode(r2d2_replay_t* r, const float* obs, const float* act, const float* rew,
                            const float* term, const float* states, int n_rows, int n_state_rows,
                            const float* priority, int n_starts, r2d2_stream_t stream);

/* One actor file at a time (LearnerReplayMemory.load, replay_memory.py:138-157): all episodes of the file are appended,
 * THEN the oldest episodes are dropped while the sequence counter exceeds max_sequences - the reference's order.
 * HOST pointers, packed over the file's episodes with R = sum(n_rows): obs [R,O], act [R,A], rew [R], term [R],
 * states [R,4,2,H] (zero rows for the pad rows), leaf_prio [R] (the priority of a row that starts a sequence, else 0).
 * Contiguous runs in the ring are one copy per tensor; the tree is refreshed once; one stream synchronisation.
 * Outputs (host, optional): first ring row of each episode, episodes evicted by this call, the sequence counter. */
int r2d2_replay_add_episodes(r2d2_replay_t* r, int n_episodes, const int* n_rows, const int* n_starts,
                             const float* obs, const float* act, const float* rew, const float* term,
                             const float* states, const float* leaf_prio, long long* row_start_out,
                             long long* n_evicted_out, long long* sequence_counter_out, r2d2_stream_t stream);

/* r2d2_replay_add_episodes plus the observation moments of the call.  obs_moments (DEVICE [1 + 2 O], or NULL for
 * r2d2_replay_add_episodes) receives (count, mean, M2) of the call's rows that are no pad row (the last n_step rows of
 * each episode, actor.py:173) and hold only finite obs values.  They are taken per ring run right after its copy -
 * a call wider than the ring overwrites its own earlier rows - in two passes (mean, then squared deviations) with
 * double partials over a fixed partition of the rows, added in a fixed order and merged run by run (Chan): the bits do
 * not depend on the schedule.  n_nonfinite_out (host, optional): the non-pad rows left out for a NaN or +-inf value.
 * Five more launches per ring run. */
int r2d2_replay_add_episodes_ex(r2d2_replay_t* r, int n_episodes, const int* n_rows, const int* n_starts,
                                const float* obs, const float* act, const float* rew, const float* term,
                                const float* states, const float* leaf_prio, long long* row_start_out,
                                long long* n_evicted_out, long long* sequence_counter_out, double* obs_moments,
                                long long* n_nonfinite_out, r2d2_stream_t stream);

/* Observation normaliser of every gather of this shard (r2d2_replay_sample, _sample_weighted, _gather and the global
 * draw's owner-side gather): the batch's obs hold x_hat of the stored raw rows (see r2d2_obs_norm_merge).  DEVICE
 * mean_f, inv_std_f [O], read at every gather (the caller keeps them alive and may rewrite them in stream order);
 * 16-byte aligned when O is a multiple of 4.  clip finite and > 0.  Both NULL: raw obs again.  The stored rows, the
 * snapshots and the export stay raw. */
int r2d2_replay_set_obs_normalizer(r2d2_replay_t* r, const float* mean_f, const float* inv_std_f, float clip);

/* Draw `batch` starts from DEVICE uniforms u[batch] in [0,1) and gather the time-major batch:
 * leaf_idx [batch] (int64, start row = tree leaf), obs [T',batch,O], act [T',batch,A], rew [T',batch],
 * term [T',batch], states [4,2,batch,H].  Any gather output may be NULL. */
int r2d2_replay_sample(r2d2_replay_t* r, const float* u, int batch, long long* leaf_idx, float* obs, float* act,
                       float* rew, float* term, float* states, r2d2_stream_t stream);

/* r2d2_replay_sample plus importance-sampling weights (prioritized replay), DEVICE is_weight [batch]:
 * is_weight[b] = (min_b' leaf_b' / leaf_b)^beta = (N P_b)^-beta / max_b' (N P_b')^-beta, leaf = the stored p^alpha,
 * normalised over this batch (the largest weight is exactly 1).  beta in [0, 1]; beta = 0 writes 1 everywhere.
 * Same draw and gather as r2d2_replay_sample, one extra single-CTA kernel. */
int r2d2_replay_sample_weighted(r2d2_replay_t* r, const float* u, int batch, float beta, long long* leaf_idx,
                                float* is_weight, float* obs, float* act, float* rew, float* term, float* states,
                                r2d2_stream_t stream);

/* The gather half alone, for start rows the caller chose (DEVICE int64 leaf_idx): same outputs as r2d2_replay_sample. */
int r2d2_replay_gather(r2d2_replay_t* r, const long long* leaf_idx, int batch, float* obs, float* act, float* rew,
                       float* term, float* states, r2d2_stream_t stream);

/* priority[leaf_idx[i]] = prio[i] (DEVICE arrays; on duplicates the highest i wins, like the python
 * loop at learner.py:136-139) and recompute the touched tree paths.  The leaf stores prio[i]^alpha under a
 * priority exponent (r2d2_replay_set_priority_exponent). */
int r2d2_replay_update_priorities(r2d2_replay_t* r, const long long* leaf_idx, const float* prio, int batch,
                                  r2d2_stream_t stream);

typedef struct {
  long long n_episodes, n_rows_used, sequence_counter, capacity_rows, tree_levels, tree_nodes;
  long long last_row_start;        /* first row of the most recently added episode */
  double total_priority;
} r2d2_replay_stats_t;
int r2d2_replay_stats(r2d2_replay_t* r, r2d2_replay_stats_t* out, r2d2_stream_t stream); /* synchronises */

/* host-side decode of a start row into the reference's (episode_index, sequence_index) pair
 * (position of the episode in FIFO order, offset inside it); -1/-1 if the row is not live. */
int r2d2_replay_decode(r2d2_replay_t* r, const long long* leaf_idx_host, int n, long long* episode_index,
                       long long* sequence_index);
/* raw device views for tests: tree level pointer/size, leaf priorities */
int r2d2_replay_tree_level(r2d2_replay_t* r, int level, const float** dev_ptr, long long* n);

/* Snapshots: a shard's whole state to the host and back (a resumed run continues bit for bit).  That state is the live
 * episodes' rows, their leaves (p^alpha; the raw priorities are not kept) and the bookkeeping below: every other leaf is
 * 0 and every tree node is the left-to-right fp32 sum of its children, so the restore rebuilds the tree from the leaves.
 * Export: r2d2_replay_export_info, the episode table in FIFO order, and any contiguous ring range of rows into HOST
 * buffers (pinned for speed) - obs [n,O], act [n,A], rew [n], term [n], states [n,4,2,H] in the STORED type (fp16 under
 * R2D2_STATE_F16), leaves [n]; plain copies, synchronises the stream.
 * Import into an EMPTY shard (else R2D2_ERR_STATE) of the same obs / act / hidden / burn-in / learning / n-step and the
 * same priority exponent (else R2D2_ERR_ARG), in three parts:
 *   begin  the snapshot's info and episode table.  Same capacity_rows: every episode goes back to its row and head is
 *          restored, so leaf indices and every tree level come back identical.  Other capacity: the episodes are
 *          compacted from row 0 in FIFO order; while they do not fit the oldest is dropped with evict_front's counter
 *          arithmetic (sequence_counter -= n_rows - (burn_in + learning), evicted_total += 1); *n_dropped_out counts them.
 *   rows   the episodes' rows packed in FIFO order (the table's order, dropped episodes included), in consecutive chunks
 *          [first, first + n), states in info->state_storage.  fp16 into an fp32 ring is widened exactly; fp32 into an
 *          fp16 ring is rounded as ingest rounds, and a finite value of magnitude >= 65520 refuses the restore.  A leaf
 *          that is negative, NaN or inf on a sequence start, or nonzero on any other row, refuses it.  Synchronises.
 *   end    checks that every row arrived, rebuilds the tree over the whole ring, commits the bookkeeping.  Synchronises.
 * Any refusal leaves the shard empty (no episode, zero counters, an all-zero tree); r2d2_last_error names the cause. */
typedef struct {
  int obs_size, n_actions, hidden, burn_in, learning, n_step;
  int state_storage;                 /* R2D2_STATE_F32 / R2D2_STATE_F16 */
  float priority_exponent;           /* alpha of the stored leaves */
  long long capacity_rows, max_sequences;
  long long n_episodes, head, sequence_counter, next_serial, evicted_total, rows_used;
} r2d2_replay_snapshot_info;
int r2d2_replay_export_info(r2d2_replay_t* r, r2d2_replay_snapshot_info* out);
/* [n_episodes] each, FIFO order */
int r2d2_replay_export_episodes(r2d2_replay_t* r, long long* row_start, int* n_rows, int* n_starts, long long* serial);
int r2d2_replay_export_rows(r2d2_replay_t* r, long long first, long long n, float* obs, float* act, float* rew,
                            float* term, void* states, float* leaves, r2d2_stream_t stream);
int r2d2_replay_import_begin(r2d2_replay_t* r, const r2d2_replay_snapshot_info* info, const long long* row_start,
                             const int* n_rows, const int* n_starts, const long long* serial, long long* n_dropped_out,
                             r2d2_stream_t stream);
int r2d2_replay_import_rows(r2d2_replay_t* r, long long first, long long n, const float* obs, const float* act,
                            const float* rew, const float* term, const void* states, const float* leaves,
                            r2d2_stream_t stream);
int r2d2_replay_import_end(r2d2_replay_t* r, r2d2_stream_t stream);

/* Global sampling over the replay shards of W data-parallel ranks (off unless a shard is attached to a group).  The W
 * shard roots form one more tree level above the shards, in rank order: global draw j of W*B takes r = u_j * total
 * (total the left-to-right fp32 sum of the roots), walks the roots as the tree walks 32 children and descends the
 * owning shard's tree with the residual; rank c trains on draws c*B .. c*B+B-1, drawn with rank c's own B uniforms.
 * At W = 1 the draw, the batch and the weights are r2d2_replay_sample(_weighted)'s bit for bit.
 * Every rank allocates `bytes` of zeroed device memory that every rank maps and attaches all W base addresses; the
 * rank's two batch slots live in that buffer (r2d2_learner_set_slot_buffers), so that the owner of a drawn row stores
 * it straight into the consumer's slot.  Every kernel runs in the caller's stream; no host synchronisation. */
typedef struct {
  size_t bytes;            /* per rank: exchange block + two batch slots */
  size_t slot_offset[2];   /* byte offset of each batch slot in the buffer */
  /* byte offsets inside a slot: obs [T,B,O], act [T,B,A], rew [T,B], term [T,B], states [4,2,B,H], leaf_idx [B]
   * (int64), shard [B] (int32), is_weight [B], uniforms [B] - every one 256-byte aligned */
  size_t off_obs, off_act, off_rew, off_term, off_states, off_leaf_idx, off_shard, off_is_weight, off_uniforms;
} r2d2_global_layout;
/* rows = burn_in + learning + n_step (host arithmetic only) */
int r2d2_global_layout_for(int rows, int batch, int obs_size, int n_actions, int hidden, int world, r2d2_global_layout* out);
/* buffer_bytes: the size every rank allocated; it must equal r2d2_global_layout_for(...).bytes of this shard's shape */
int r2d2_replay_attach_group(r2d2_replay_t* r, int rank, int world, int batch, void* const* peer_bases,
                             size_t buffer_bytes);
/* Write-back of the batch this rank trained on: DEVICE leaf_idx [B], shard [B] (its slot's), raw priority [B].  Stage 0
 * publishes the B records to every rank, stage 1 waits for every rank's records and applies those of this shard in
 * global-index order (the highest index wins on a duplicate leaf); -1 runs both.  Must alternate with draws. */
int r2d2_replay_global_write_back(r2d2_replay_t* r, int stage, const long long* leaf_idx, const int* shard,
                                  const float* priority, r2d2_stream_t stream);
/* Draw the next batch into batch slot `slot` (its uniforms [B] hold this rank's draws).  Stage 0 publishes this shard's
 * root (after the write-back and any ingest) and the uniforms, stage 1 waits for every root, draws, gathers this
 * shard's rows into the consumers' slots and signals delivery with the minimum drawn leaf, stage 2 waits for every
 * owner's delivery and, with `weighted`, turns the leaf values into (min / leaf)^beta over the global batch; -1 runs
 * all three.  7 kernels per iteration with the write-back (2 + 5). */
int r2d2_replay_global_draw(r2d2_replay_t* r, int stage, int slot, int weighted, float beta, r2d2_stream_t stream);
/* 0 = fine, 1 = a bounded wait (4 s) for a peer's flag expired (synchronises the stream) */
int r2d2_replay_global_status(r2d2_replay_t* r, int* status, r2d2_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Learner iteration engine (learner.py:84-139 minus file I/O).  Parameters, gradients and Adam
 * moments are caller-owned flat device buffers; the engine owns batch buffers and workspaces.
 * ---------------------------------------------------------------------------------------------- */
typedef struct r2d2_learner r2d2_learner_t;

typedef struct {
  int obs_size, n_actions, hidden;
  int batch, burn_in, learning, n_step;
  float gamma, actor_lr, critic_lr, eta;
  int target_update_interval;      /* learner.py:45,131 */
  float* actor_params;  float* critic_params;  float* target_actor_params;  float* target_critic_params;
  float* actor_grads;   float* critic_grads;
  float* actor_exp_avg; float* actor_exp_avg_sq; float* critic_exp_avg; float* critic_exp_avg_sq;
} r2d2_learner_config;

typedef struct {
  /* device pointers into the engine-owned batch (fill them via r2d2_replay_sample or memcpy) */
  float* obs;      /* [T',B,O] */
  float* act;      /* [T',B,A] */
  float* rew;      /* [T',B]   */
  float* term;     /* [T',B]   */
  float* states;   /* [4,2,B,H] actor, target_actor, critic, target_critic */
  long long* leaf_idx; /* [B] */
  float* uniforms; /* [B] */
  /* results of the last iteration */
  float* q_value;        /* [L,B,A] */
  float* target_q_value; /* [L,B,A] */
  float* td_sq;          /* [L,B]   */
  float* priority;       /* [B]     */
  float* losses;         /* [2] critic_loss, actor_loss; [3] with the twin critic: critic 2's loss in [2] */
} r2d2_learner_buffers;

int r2d2_learner_create(r2d2_learner_t** out, const r2d2_learner_config* cfg);
int r2d2_learner_destroy(r2d2_learner_t* l);

/* TD3's target (Fujimoto et al. 2018; delayed policy updates are not part of it here), off by default.
 *
 * twin_critic (create-time: it sizes the buffers and the arena).  With it on, EVERY critic_* pointer of the config -
 * critic_params, target_critic_params, critic_grads, critic_exp_avg, critic_exp_avg_sq - is a block of 2 P' floats
 * [critic 1 | pad | critic 2 | pad], P the critic's parameter count and P' = P rounded up to a multiple of 64 floats
 * (critic 2 starts at float P', 256-byte aligned like critic 1: the GEMM kernels read weights with vector loads).  The
 * padding is zero and stays zero (zero gradients, zero moments).  Then:
 *   - y is today's target (rescaling, options and weights included) with q' = min(Q'_1(s, a'), Q'_2(s, a')) elementwise;
 *     both rescalings are monotone, so the minimum of the raw outputs is the minimum after h_eps^-1;
 *   - each critic's loss is today's MSE against y, each gets its own BPTT into its half of critic_grads;
 *   - critic 1 is the existing critic: it alone starts from the stored recurrent state (states[2] / states[3]), it alone
 *     feeds the DPG actor loss, the priorities, td_sq and target_q_value.  Critic 2 and its target start from the zero
 *     state and rely on the burn-in rows: the replay's states[4,2,B,H] carry the four reference nets only;
 *   - Adam over the 2 P block is two independent Adams with one lr and step; gradient-norm clipping is JOINT over both
 *     critics (clip_grad_norm_ over the twin module), and the critic norm of r2d2_learner_grad_norms is that joint norm;
 *     the hard copy, the Polyak blend and the data-parallel exchange cover the whole block.
 * NULL options = r2d2_learner_create. */
typedef struct {
  int twin_critic;   /* 0 or 1 */
} r2d2_learner_options;
int r2d2_learner_create_ex(r2d2_learner_t** out, const r2d2_learner_config* cfg, const r2d2_learner_options* options);
/* Target policy smoothing: a' = clip(mu'(s) + clip(sigma z, -clip, clip), -1, 1) on the target actor's actions of the
 * rows the target critic bootstraps from (rows [Bn+n, Bn+n+L) of its input; the stored actions before them are
 * untouched); every target critic sees the same a'.  z comes from r2d2_target_smoothing's generator with key (seed, rank)
 * and iter = the index of the iteration that trains on the batch (critic phases run so far; r2d2_learner_set_step_count
 * sets it too), so a pipelined, a sequential and a resumed run draw the same noise.  sigma = 0 (the default) is off: no
 * launch.  sigma finite >= 0 and clip finite > 0, else R2D2_ERR_ARG; R2D2_ERR_STATE while a target phase has run
 * ahead and not yet been consumed by a critic phase. */
int r2d2_learner_set_target_smoothing(r2d2_learner_t* l, float sigma, float clip, unsigned int seed, unsigned int rank);
/* DEVICE address of critic 2's q [L,B,A] (NULL without the twin), critic 2's offset P' in floats inside each critic
 * block (0 without the twin) and the arena bytes the twin added (0 without it).  Critic 2's loss is losses[2] of
 * r2d2_learner_buffers. */
int r2d2_learner_twin_buffers(r2d2_learner_t* l, float** q2, long long* critic2_offset, size_t* twin_bytes);
/* The smoothing kernel alone: out[e] = clip(mu[e] + clip(sigma z_e, -clip, clip), -1, 1), e < n (out may be mu).
 * z_e: Philox4x32-10 with key = (seed, rank), counter = (e >> 2, (uint32) iter, iter >> 32, 0); the output words
 * (x0, x1) serve e % 4 in {0, 1} and (x2, x3) serve {2, 3}; u = (2 (x >> 9) + 1) 2^-24; z = sqrt(-2 ln u_a) cos(2 pi u_b)
 * for the even element of a pair and sin for the odd one, (u_a, u_b) the pair's two words, in fp32 with precise logf,
 * sqrtf and sincospif.  One launch. */
int r2d2_target_smoothing(const float* mu, float* out, long long n, float sigma, float clip, unsigned int seed,
                          unsigned int rank, unsigned long long iter, r2d2_stream_t stream);
int r2d2_learner_buffers_get(r2d2_learner_t* l, r2d2_learner_buffers* out);
/* The batch has two slots.  r2d2_learner_buffers_get returns slot 0 (the only one a simple caller needs); a pipelined
 * caller fills slot 1-s with batch i+1 while the phases of iteration i still read slot s, runs that batch's target
 * chains early with r2d2_learner_target_phase (they read only the target nets: learner.py:87,94-95,106) and switches
 * with r2d2_learner_select_batch before the next r2d2_learner_critic_phase.  Not allowed on an iteration that updates
 * the target nets (step count + 1 a multiple of target_update_interval) from its actor phase until its finish phase:
 * with target_tau < 1 the actor phase already blends the critic's target, and the finish phase updates the actor's
 * target (or copies both at target_tau = 1) - target chains run in between would read stale targets. */
int r2d2_learner_buffers_get_slot(r2d2_learner_t* l, int slot, r2d2_learner_buffers* out);
int r2d2_learner_select_batch(r2d2_learner_t* l, int slot);
/* Importance weights of a batch slot: [B] floats next to leaf_idx / uniforms (fill them with
 * r2d2_replay_sample_weighted or memcpy; 1 after create).  The critic phase reads the selected slot's weights only
 * while importance weighting is on; off (the default) it runs the unweighted TD kernels. */
int r2d2_learner_is_weights(r2d2_learner_t* l, int slot, float** out);
/* Move batch slot `slot` into caller-owned device memory (global sampling: the slots in the buffer every rank maps):
 * obs .. uniforms of `b` (the other fields are ignored) and is_weight [B].  Refused while a prefetched batch's target
 * chains are pending; the default slots stay allocated in the learner's arena. */
int r2d2_learner_set_slot_buffers(r2d2_learner_t* l, int slot, const r2d2_learner_buffers* b, float* is_weight);
int r2d2_learner_set_importance_weighting(r2d2_learner_t* l, int on);
/* Polyak target update (utils.py:4-6): on the iterations of the hard copy (step % target_update_interval == 0) each
 * target becomes fl(fl(target * (float)(1 - (double)tau)) + fl(param' * tau)), param' the net's post-Adam weight, fused
 * into that net's Adam launch (critic: actor phase, actor: finish phase).  tau in (0, 1]; 1 (the default) is the hard
 * copy, unchanged.  Anything else, NaN included, is R2D2_ERR_ARG. */
int r2d2_learner_set_target_tau(r2d2_learner_t* l, float tau);
/* Global gradient-norm clipping per net (torch.nn.utils.clip_grad_norm_ over the whole flat block): with
 * g = grads * grad_scale, N = ||g||_2 and c = min(1, max_norm / (N + 1e-6)), Adam consumes fl(g * c).  One norm kernel
 * before each Adam, no host synchronisation, no floating-point atomics.  0 (the default) = off, no kernel; negative,
 * NaN or inf is R2D2_ERR_ARG. */
int r2d2_learner_set_grad_clip(r2d2_learner_t* l, float max_norm);
/* The learner's n-step target and priority options (r2d2_td_options; the defaults after create).  Either may change between
 * any two iterations: q_next is the target critic's raw output in every mode, h_eps^-1 is applied inside the TD kernel.
 * Same kernel count per iteration in every combination.  Bad values are R2D2_ERR_ARG and leave the setting as it was. */
int r2d2_learner_set_value_rescaling(r2d2_learner_t* l, int mode, float eps);
int r2d2_learner_set_priority_metric(r2d2_learner_t* l, int metric);
/* DEVICE address of [critic N, actor N], the pre-clip norms of the last optimiser steps (written only while clipping
 * or metrics are on; 0 after create) */
int r2d2_learner_grad_norms(r2d2_learner_t* l, float** out);
int r2d2_learner_target_phase(r2d2_learner_t* l, int slot, r2d2_stream_t stream);
/* forget a target phase that ran ahead: the caller is about to overwrite that slot's batch */
int r2d2_learner_discard_prefetch(r2d2_learner_t* l, r2d2_stream_t stream);
/* phase 1: target chains (unless r2d2_learner_target_phase already ran for the selected slot), online critic chain,
 * TD/priority kernel, critic BPTT -> critic_grads.  On one GPU (no peers attached, actor-input overlap on) and unless
 * R2D2_OVERLAP_INPUTS=0, whole chains run on a second stream the learner owns: the actor's forward chain from the start
 * of this call, and everything after the TD kernels (critic BPTT, the twin's chain, TD and BPTT, the metrics record).
 * The priorities, q, target and losses[0] are ordered on `stream` when this call returns; critic_grads, losses[2] and the
 * metrics record only after r2d2_learner_actor_phase (or r2d2_learner_discard_prefetch) on that stream. */
int r2d2_learner_critic_phase(r2d2_learner_t* l, r2d2_stream_t stream);
/* optional, between phase 1 and phase 2: the actor's forward chain of the DPG update (learner.py:117,120-123; zero
 * state, 2 cell steps per row).  It does not read the critic, so a data-parallel caller issues it while the
 * all-reduce of critic_grads is in flight; phase 2 then skips it.  Without this call phase 2 runs it itself.  A no-op
 * when it already ran for the iteration (phase 1 issues it on the second stream, see above). */
int r2d2_learner_actor_forward(r2d2_learner_t* l, r2d2_stream_t stream);
/* phase 2: critic Adam (grads * grad_scale; norm kernel first when clipping, Polyak update of the critic's target on
 * update iterations when target_tau < 1), actor chain unless r2d2_learner_actor_forward already ran, critic on actor
 * actions, dgrad through critic, actor BPTT -> actor_grads */
int r2d2_learner_actor_phase(r2d2_learner_t* l, float grad_scale, r2d2_stream_t stream);
/* phase 3: actor Adam (same extras as the critic's), step counter, hard target update every target_update_interval
 * steps at target_tau = 1 */
int r2d2_learner_finish_phase(r2d2_learner_t* l, float grad_scale, r2d2_stream_t stream);
int r2d2_learner_step_count(r2d2_learner_t* l);
/* The critic phase pre-issues the input projection of the actor's DPG chain on a side stream (it reads the actor's
 * weights).  A caller that runs phase 3 of iteration i AFTER phase 1 of iteration i+1 (deferred actor all-reduce)
 * switches that off: the weights are not final yet. */
int r2d2_learner_set_overlap_actor_inputs(r2d2_learner_t* l, int on);
/* Data-parallel learner, one process per GPU (SURVEY 8e): the two gradient all-reduces of learner.py:113-114,127-128
 * as kernels of this library over NVLink peer memory, issued inside the phases on the learner's own stream (peer.cuh).
 * Every rank allocates `bytes` of zeroed device memory that all ranks of the node can map (CUDA IPC / fabric handles;
 * the Python host side uses torch's symmetric memory), exchanges the addresses and attaches them; the learner's
 * gradient blocks then live at off_*_grads of its own buffer and the optimiser kernels read off_*_sums.  The caller
 * keeps calling the phases in the same order on every rank and passes grad_scale = 1 / world.  Call order with the
 * loosest coupling: critic_phase(i), finish_phase(i-1), actor_forward(i), actor_phase(i). */
typedef struct {
  size_t bytes, off_critic_grads, off_actor_grads, off_critic_sums, off_actor_sums;
} r2d2_peer_layout;
int r2d2_learner_peer_layout(r2d2_learner_t* l, int world, r2d2_peer_layout* out);
/* the same from the two parameter counts (host arithmetic only) */
int r2d2_peer_layout_for(long long n_critic, long long n_actor, int world, r2d2_peer_layout* out);
int r2d2_learner_attach_peers(r2d2_learner_t* l, int rank, int world, void* const* peer_bases);
/* 0 = fine, 1 = a bounded wait (4 s) for a peer expired: the replicas are no longer in step (synchronises the stream) */
int r2d2_learner_peer_status(r2d2_learner_t* l, int* status, r2d2_stream_t stream);
/* diagnostics: nanoseconds summed since the last reset - [0..1] the slice-sum kernel waited for the peers' "gradients
 * complete" (critic, actor block), [2..3] the slice-sum kernel ran in total, [4..5] the wait kernel waited */
int r2d2_learner_peer_counters(r2d2_learner_t* l, unsigned long long* out6, int reset, r2d2_stream_t stream);
/* resume: completed iterations so far (drives Adam's bias correction and the target-update period, learner.py:82,131) */
int r2d2_learner_set_step_count(r2d2_learner_t* l, int step);
/* Learner metrics, off by default: one record of r2d2_metrics_field_count() doubles per learner iteration, reduced on
 * the device in the learner's stream - no host synchronisation - into a caller-owned device ring of `slots` records.
 * Iteration i (the step count at its critic phase, so a resumed run continues the numbering) writes record i % slots.
 * Fields, in order (r2d2_metrics_field_name(k) gives each name):
 *    0 iteration         i: marks which iteration owns the slot
 *    1 t_ns              %globaltimer when the critic phase's metrics kernel runs (differences: the iteration period;
 *                        held in a double, so in steps of 256 ns at today's epoch times)
 *    2 critic_loss       losses[0]
 *    3 critic2_loss      losses[2] with the twin critic, else NaN
 *    4 actor_loss        losses[1]
 *    5-7 q_mean, q_min, q_max                  over critic 1's q [L,B,A]
 *    8-10 target_mean, target_min, target_max  over the TD target y [L,B,A]
 *    11-12 td_abs_mean, td_abs_max             |q - y| formed in double
 *    13-14 priority_mean, priority_max         the raw priorities written back [B]
 *    15-16 is_weight_min, is_weight_mean       the importance weights [B]; both 1 with importance weighting off
 *    17 q2_mean          critic 2's q with the twin critic, else NaN
 *    18 mu_abs_mean      mean |mu| over the actor head's output [L,B,A]
 *    19 mu_saturated     the fraction of mu with |mu| >= 0.99
 *    20 critic_grad_norm the pre-clip L2 norm of the gradient the critic's Adam consumed (grad_scale applied: the rank
 *                        mean in data-parallel runs), as r2d2_learner_grad_norms; twin: joint over both critics
 *    21 actor_grad_norm  the same for the actor.  It exists only after the finish phase, which in data-parallel runs
 *                        follows the next critic phase: the device record holds NaN, and the finish phase copies the
 *                        float norm into float k of the side array behind the records (k = the iteration's slot)
 *    22 nonfinite        count of NaN / +-inf in q, y, q2 and mu
 * Means are sums in double over the element count; min / max skip NaN (they are counted in nonfinite).  Fields 0-3, 5-17
 * and 22 are written at the end of the critic phase, 4 and 18-20 (and 22's mu count) in the actor phase.  Sums are
 * added in a fixed order and no floating-point atomic is used: two seeded runs write the same bits.  A record is
 * complete once its iteration's finish phase has run.
 *
 * Switching metrics on adds per iteration one kernel to the critic phase and one to the actor phase, and - without
 * gradient-norm clipping - the norm kernel before each Adam (r2d2_learner_grad_norms is then written too): 4 launches,
 * 2 with clipping on.  Training is unchanged bit for bit; off (the default) issues none of it.
 *
 * ring: r2d2_metrics_ring_bytes(slots) bytes of device memory, 8-byte aligned - slots * fields doubles of records
 * followed by slots floats of actor norms - or NULL to switch metrics off.  slots >= 1, else R2D2_ERR_ARG.  Only before
 * the learner's first critic phase, else R2D2_ERR_STATE. */
size_t r2d2_metrics_ring_bytes(int slots);
int r2d2_metrics_field_count(void);
const char* r2d2_metrics_field_name(int field);   /* NULL outside [0, r2d2_metrics_field_count()) */
int r2d2_learner_set_metrics(r2d2_learner_t* l, void* ring, int slots);
/* number of kernels launched by the three phases of one iteration (bench.py's gpu_launches) */
int r2d2_learner_launches_per_iteration(r2d2_learner_t* l);

#ifdef __cplusplus
}
#endif
#endif /* R2D2_B200_H_ */

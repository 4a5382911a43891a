// r2d2_policy_step: one env step of the four recurrent nets of N actor lanes (Actor.run, actor.py:149-154):
//
//   mu   = tanh(l3(tanh(h'))),  (h', c') = LSTMCell(tanh(l1(obs)), (h, c))           actor, target actor
//   (h', c') = LSTMCell(tanh(l1(cat(obs, mu))), (h, c))                               critic (target critic: mu_t)
//
// The critics' heads are discarded by the reference and are not computed.  Five launches, one per phase of the
// dependency chain, each chained to the one before with programmatic dependent launch:
//
//   1. every net:    G = W_hh h + (b_ih + b_hh);  actors: Z = tanh(W1 obs + b1);  critics: Z = W1[:, :O] obs + b1
//   2. actor cells:  gates = W_ih Z + G -> (h', c')                                         nets 0, 1
//   3. heads:        mu = tanh(W3 tanh(h') + b3), mu_t likewise                              nets 0, 1
//   4. critic l1:    Z = tanh(W1[:, O:] mu + Z)   (target critic: mu_t), in place            nets 2, 3
//   5. critic cells: as phase 2                                                             nets 2, 3
//
// Work unit: one warp computes 4 weight rows for a tile of 16 lanes.  Weights are read straight from the flat
// state_dict blocks (row-major [out, in]); lane l of the warp takes k = l, l + 32, ... of every row, so a row read is
// one 128-byte line per 32 k.  The 16 lanes' inputs are staged in shared memory k-major ([k][16 + 4 pad]), one float4
// per 4 lanes.  After the k loop a 5-round butterfly reduce-scatter leaves each of the 32 threads with 2 of the 64
// (row, lane) sums.  The cell phases take the 4 gate rows of one hidden unit, so the pointwise update needs only
// shuffles.
//
// Determinism: every output element is summed in the same order whatever N is and wherever its lane sits in a tile
// (per thread k ascending, then the same butterfly tree), with no atomics, so lane n's bits do not depend on the
// other lanes.
//
// Exploration (r2d2_policy_step_explore): phase 3 runs as policy_explore_head_kernel, which also turns each of the
// actor's mu elements into its noisy action from the same registers (explore_action).  The other four phases and mu
// itself are unchanged.
//
// Each kernel issues L2 prefetches of its weight rows before griddepcontrol.wait, so they overlap the tail of the
// phase before; every kernel executes the wait, which makes the chain transitive (phase 5 may read phase 1's G).
#include <cmath>
#include <vector>

#include "obs_norm.cuh"
#include "philox.cuh"
#include "policy.cuh"

namespace r2d2 {
namespace {

constexpr int NT = 16;             // lanes per tile
constexpr int XS = NT + 4;         // staged row stride in floats: conflict-free float4 reads for 8 consecutive k
constexpr int KC = 512;            // k per staged chunk
constexpr int WARPS = 8;
constexpr int THREADS = WARPS * 32;

struct StepArgs {
  const float *p0, *p1, *p2, *p3;  // actor, target actor, critic, target critic
  const float* obs;                // [N,O]
  const float* state_in;           // [4,2,N,H]
  float* state_out;                // [4,2,N,H]
  float* mu;                       // [N,A]
  float* G;                        // [4,N,4H] W_hh h + b_ih + b_hh
  float* Z;                        // [4,N,H]  l1 outputs (critics: obs half until phase 4)
  float* mu_t;                     // [N,A]
  int N, O, A, H;
  const float *obs_mean, *obs_inv_std;   // r2d2_policy_step_ex: phase 1 stages obs_norm_apply(obs) (the kNorm kernel)
  float obs_clip;
};

// r2d2_exploration as the head kernel reads it
struct ExploreArgs {
  const unsigned int* actor_id;    // [N]
  const float* sigma;              // [N]
  float* ou_state;                 // [N,A] (OU)
  float* action;                   // [N,A]
  uint32_t seed, step_lo, step_hi;
  float one_minus_theta;
};

constexpr int kNoNoise = 0, kGaussian = 1, kOU = 2;

struct NetView {
  const float *w1, *b1, *wih, *whh, *bih, *bhh, *w3, *b3;
  int I;
};

__device__ __forceinline__ NetView net_view(const StepArgs& a, int net) {
  const float* p = net == 0 ? a.p0 : net == 1 ? a.p1 : net == 2 ? a.p2 : a.p3;
  const int I = a.O + (net >= 2 ? a.A : 0);
  const size_t H = a.H;
  NetView v;
  v.I = I;
  v.w1 = p;                 v.b1 = v.w1 + H * I;
  v.wih = v.b1 + H;         v.whh = v.wih + 4 * H * H;
  v.bih = v.whh + 4 * H * H; v.bhh = v.bih + 4 * H;
  v.w3 = v.bhh + 4 * H;     v.b3 = v.w3 + (size_t)a.A * H;
  return v;
}

__device__ __forceinline__ float sigmoid_acc(float x) { return 1.0f / (1.0f + expf(-x)); }

__device__ __forceinline__ void prefetch_rows(const float* const (&w)[4], int K) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int r = 0; r < 4; ++r)
    for (int k = lane * 32; k < K; k += 32 * 32)
      asm volatile("prefetch.global.L2 [%0];" ::"l"(w[r] + k));
}

// xs[k][n] = src[n*ld + k] (tanh'd if kTanh; kNorm: obs_norm_apply with mean[k], inv_std[k]) for k < kc, n < nl;
// zero for nl <= n < NT
template <bool kTanh, bool kNorm = false>
__device__ __forceinline__ void stage(float* xs, const float* src, long long ld, int kc, int nl,
                                      const float* mean = nullptr, const float* inv_std = nullptr, float clip = 0.f) {
  for (int i = threadIdx.x; i < NT * kc; i += THREADS) {
    const int n = i / kc, k = i - n * kc;
    float x = 0.0f;
    if (n < nl) {
      x = src[(long long)n * ld + k];
      if (kTanh) x = tanhf(x);
      if (kNorm) x = obs_norm_apply(x, __ldg(mean + k), __ldg(inv_std + k), clip);
    }
    xs[k * XS + n] = x;
  }
}

// one round of the reduce-scatter over the first 4*O live values: O = 16, 8, 4, 2, 1.  A compile-time O keeps every
// index constant, so the accumulators stay in registers.
template <int O>
__device__ __forceinline__ void reduce_round(float (&acc)[4 * NT], int lane) {
  constexpr int HALF = 2 * O;
  const bool up = (lane & O) != 0;
#pragma unroll
  for (int i = 0; i < HALF; ++i) {
    const float send = up ? acc[i] : acc[i + HALF];
    const float keep = up ? acc[i + HALF] : acc[i];
    acc[i] = keep + __shfl_xor_sync(0xffffffffu, send, O);
  }
}

// v[i] = sum_k w[r][k] * x[n][k] for (r, n) = (lane / 8, 2 * (lane % 8) + i), x = src[n*ld + k] over the tile's
// nl lanes.  Block-uniform K and src: every warp of the block calls it.
template <bool kTanh, bool kNorm = false>
__device__ __forceinline__ void rows_dot(float (&v)[2], const float* const (&w)[4], int K, const float* src,
                                         long long ld, int nl, float* xs, const float* mean = nullptr,
                                         const float* inv_std = nullptr, float clip = 0.f) {
  const int lane = threadIdx.x & 31;
  float acc[4 * NT];
#pragma unroll
  for (int i = 0; i < 4 * NT; ++i) acc[i] = 0.0f;
  for (int k0 = 0; k0 < K; k0 += KC) {
    const int kc = min(KC, K - k0);
    __syncthreads();                                   // the previous chunk is consumed
    if (kNorm) stage<kTanh, true>(xs, src + k0, ld, kc, nl, mean + k0, inv_std + k0, clip);
    else stage<kTanh>(xs, src + k0, ld, kc, nl);
    __syncthreads();
#pragma unroll 2
    for (int k = lane; k < kc; k += 32) {
      float wv[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) wv[r] = __ldg(w[r] + k0 + k);
      const float4* xp = reinterpret_cast<const float4*>(xs + k * XS);
      float x[NT];
#pragma unroll
      for (int q = 0; q < NT / 4; ++q) {
        const float4 t = xp[q];
        x[4 * q] = t.x; x[4 * q + 1] = t.y; x[4 * q + 2] = t.z; x[4 * q + 3] = t.w;
      }
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int n = 0; n < NT; ++n) acc[r * NT + n] = fmaf(wv[r], x[n], acc[r * NT + n]);
    }
  }
  // butterfly reduce-scatter: each round halves the live values; the thread with bit O set keeps the upper half.
  // Thread t ends with flat indices 2t, 2t + 1 (flat = r * NT + n).
  reduce_round<16>(acc, lane);
  reduce_round<8>(acc, lane);
  reduce_round<4>(acc, lane);
  reduce_round<2>(acc, lane);
  reduce_round<1>(acc, lane);
  v[0] = acc[0];
  v[1] = acc[1];
}

// LSTM cell of hidden unit j for the tile's lanes: thread t < NT takes lane t; gate r of lane t sits in thread
// 8r + t/2, slot t&1 (rows_dot's layout).
__device__ __forceinline__ void cell_update(const float (&v)[2], const StepArgs& a, int net, int j, int tile0) {
  const int lane = threadIdx.x & 31;
  const int t = lane & (NT - 1);
  float pre[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const float a0 = __shfl_sync(0xffffffffu, v[0], 8 * r + (t >> 1));
    const float a1 = __shfl_sync(0xffffffffu, v[1], 8 * r + (t >> 1));
    pre[r] = (t & 1) ? a1 : a0;
  }
  const int n = tile0 + t;
  if (lane >= NT || n >= a.N) return;
  const size_t H = a.H, N = a.N;
  const float* g = a.G + ((size_t)net * N + n) * 4 * H;
  const float gi = sigmoid_acc(pre[0] + g[j]);
  const float gf = sigmoid_acc(pre[1] + g[H + j]);
  const float gg = tanhf(pre[2] + g[2 * H + j]);
  const float go = sigmoid_acc(pre[3] + g[3 * H + j]);
  const float c = a.state_in[((size_t)(net * 2 + 1) * N + n) * H + j];
  const float c2 = gf * c + gi * gg;
  a.state_out[((size_t)(net * 2 + 1) * N + n) * H + j] = c2;
  a.state_out[((size_t)(net * 2) * N + n) * H + j] = go * tanhf(c2);
}

// lane n's action a from its noise-free mu m (include/r2d2_b200.h r2d2_exploration); under OU x is updated in place
template <int kNoise>
__device__ __forceinline__ float explore_action(const ExploreArgs& e, float m, int n, int a, int A) {
  const Philox4 r = philox4x32_10((uint32_t)(a >> 2), e.step_lo, e.step_hi, 1u, e.seed, __ldg(e.actor_id + n));
  const bool upper = (a & 2) != 0;                    // words (x2, x3) serve a % 4 in {2, 3}
  float rad, s, c;
  box_muller(upper ? r.x[2] : r.x[0], upper ? r.x[3] : r.x[1], rad, s, c);
  const float z = __fmul_rn(rad, (a & 1) ? s : c);
  float noise = __fmul_rn(__ldg(e.sigma + n), z);
  if (kNoise == kOU) {
    float* x = e.ou_state + (size_t)n * A + a;
    noise = __fadd_rn(__fmul_rn(e.one_minus_theta, *x), noise);
    *x = noise;
  }
  return fminf(fmaxf(__fadd_rn(m, noise), -1.0f), 1.0f);
}

__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;"); }

// kNormObs (phase 1 only): the obs rows are normalised as they are staged.  kNoise (phase 3 only): the actor head
// also writes e.action.
template <int PHASE, bool kNormObs, int kNoise = kNoNoise>
__device__ __forceinline__ void policy_phase(const StepArgs& a, const ExploreArgs& e = ExploreArgs{}) {
  __shared__ __align__(16) float xs[KC * XS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile0 = blockIdx.y * NT;
  const int nl = min(NT, a.N - tile0);
  const int H = a.H, N = a.N;
  float v[2];
  const int r_out = lane >> 3;                         // row of this thread's two sums
  const int n_out = tile0 + 2 * (lane & 7);            // lane of v[0]; v[1] is the next one

  if (PHASE == 1) {
    const int net = blockIdx.z;
    const NetView P = net_view(a, net);
    const int n_whh_blocks = H / WARPS;
    if ((int)blockIdx.x < n_whh_blocks) {             // W_hh h: the 4 gate rows of hidden unit j
      const int j = blockIdx.x * WARPS + warp;
      const float* w[4] = {P.whh + (size_t)j * H, P.whh + (size_t)(H + j) * H, P.whh + (size_t)(2 * H + j) * H,
                           P.whh + (size_t)(3 * H + j) * H};
      prefetch_rows(w, H);
      pdl_wait();
      pdl_launch_dependents();
      rows_dot<false>(v, w, H, a.state_in + ((size_t)(net * 2) * N + tile0) * H, H, nl, xs);
      const int row = r_out * H + j;
      const float b = P.bih[row] + P.bhh[row];
#pragma unroll
      for (int i = 0; i < 2; ++i)
        if (n_out + i < N) a.G[((size_t)net * N + n_out + i) * 4 * H + row] = v[i] + b;
    } else {                                          // W1 obs: rows 4q .. 4q+3 (critics: the obs columns)
      const int q = (blockIdx.x - n_whh_blocks) * WARPS + warp;
      const float* w[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) w[r] = P.w1 + (size_t)(4 * q + r) * P.I;
      prefetch_rows(w, a.O);
      pdl_wait();
      pdl_launch_dependents();
      if (kNormObs)
        rows_dot<false, true>(v, w, a.O, a.obs + (size_t)tile0 * a.O, a.O, nl, xs, a.obs_mean, a.obs_inv_std, a.obs_clip);
      else
        rows_dot<false>(v, w, a.O, a.obs + (size_t)tile0 * a.O, a.O, nl, xs);
      const int row = 4 * q + r_out;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const float z = v[i] + P.b1[row];
        if (n_out + i < N) a.Z[((size_t)net * N + n_out + i) * H + row] = net < 2 ? tanhf(z) : z;
      }
    }
  } else if (PHASE == 2 || PHASE == 5) {              // cells: W_ih z + G
    const int net = blockIdx.z + (PHASE == 5 ? 2 : 0);
    const NetView P = net_view(a, net);
    const int j = blockIdx.x * WARPS + warp;
    const float* w[4] = {P.wih + (size_t)j * H, P.wih + (size_t)(H + j) * H, P.wih + (size_t)(2 * H + j) * H,
                         P.wih + (size_t)(3 * H + j) * H};
    prefetch_rows(w, H);
    pdl_wait();
    pdl_launch_dependents();
    rows_dot<false>(v, w, H, a.Z + ((size_t)net * N + tile0) * H, H, nl, xs);
    cell_update(v, a, net, j, tile0);
  } else if (PHASE == 3) {                            // heads: mu = tanh(W3 tanh(h') + b3)
    const int net = blockIdx.z;
    const NetView P = net_view(a, net);
    const int q = blockIdx.x * WARPS + warp;
    const float* w[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) w[r] = P.w3 + (size_t)min(4 * q + r, a.A - 1) * H;
    prefetch_rows(w, H);
    pdl_wait();
    pdl_launch_dependents();
    rows_dot<true>(v, w, H, a.state_out + ((size_t)(net * 2) * N + tile0) * H, H, nl, xs);
    const int row = 4 * q + r_out;
    float* out = net == 0 ? a.mu : a.mu_t;
    if (row < a.A) {
#pragma unroll
      for (int i = 0; i < 2; ++i)
        if (n_out + i < N) {
          const float m = tanhf(v[i] + P.b3[row]);
          out[(size_t)(n_out + i) * a.A + row] = m;
          if (kNoise != kNoNoise && net == 0)
            e.action[(size_t)(n_out + i) * a.A + row] = explore_action<kNoise>(e, m, n_out + i, row, a.A);
        }
    }
  } else {                                            // PHASE 4: critics' action columns of l1, then tanh
    const int net = 2 + blockIdx.z;
    const NetView P = net_view(a, net);
    const int q = blockIdx.x * WARPS + warp;
    const float* w[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) w[r] = P.w1 + (size_t)(4 * q + r) * P.I + a.O;
    prefetch_rows(w, a.A);
    pdl_wait();
    pdl_launch_dependents();
    rows_dot<false>(v, w, a.A, (net == 2 ? a.mu : a.mu_t) + (size_t)tile0 * a.A, a.A, nl, xs);
    const int row = 4 * q + r_out;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      if (n_out + i < N) {
        float* z = a.Z + ((size_t)net * N + n_out + i) * H + row;
        *z = tanhf(v[i] + *z);
      }
    }
  }
}

template <int PHASE>
__global__ void __launch_bounds__(THREADS, 2) policy_phase_kernel(const StepArgs a) {
  policy_phase<PHASE, false>(a);
}

// phase 1 of r2d2_policy_step_ex with an observation normaliser
__global__ void __launch_bounds__(THREADS, 2) policy_obs_norm_phase1_kernel(const StepArgs a) {
  policy_phase<1, true>(a);
}

// phase 3 of r2d2_policy_step_explore (kNoise: kGaussian or kOU)
template <int kNoise>
__global__ void __launch_bounds__(THREADS, 2) policy_explore_head_kernel(const StepArgs a, const ExploreArgs e) {
  policy_phase<3, false, kNoise>(a, e);
}

template <typename Kernel, typename... Extra>
int launch_phase(Kernel kernel, dim3 grid, const StepArgs& a, cudaStream_t stream, const Extra&... extra) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = dim3(THREADS);
  cfg.dynamicSmemBytes = 0;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  R2D2_CUDA_TRY(cudaLaunchKernelEx(&cfg, kernel, a, extra...));
  count_launch();
  return R2D2_OK;
}

}  // namespace

size_t policy_workspace_floats(int O, int A, int H, int N) {
  (void)O;
  return (size_t)N * H * 16 + (size_t)N * H * 4 + (size_t)N * A;
}

int policy_step(int O, int A, int H, const float* const params[4], const float* obs, const float* state_in,
                float* state_out, float* mu, int N, float* workspace, cudaStream_t stream, const float* obs_mean,
                const float* obs_inv_std, float obs_clip, const r2d2_exploration* explore, float* action) {
  R2D2_REQUIRE(params && params[0] && params[1] && params[2] && params[3] && obs && state_in && state_out && mu &&
                   workspace, "null");
  R2D2_REQUIRE(state_in != state_out, "state_in and state_out must be different buffers");
  R2D2_REQUIRE((obs_mean == nullptr) == (obs_inv_std == nullptr), "obs_mean and obs_inv_std are both given or both NULL");
  R2D2_REQUIRE(!obs_mean || (obs_clip > 0.f && obs_clip <= 3.402823466e38f), "clip must be finite and > 0");
  if (N < 1 || N > kPolicyMaxLanes || H < 32 || H > kPolicyMaxHidden || H % 32 != 0 || A < 1 ||
      A > kPolicyMaxActions || O < 1) {
    set_last_error("r2d2_policy_step: unsupported shape N=" + std::to_string(N) + " O=" + std::to_string(O) +
                   " A=" + std::to_string(A) + " H=" + std::to_string(H) + " (supported: 1 <= N <= " +
                   std::to_string(kPolicyMaxLanes) + ", H a multiple of 32 up to " + std::to_string(kPolicyMaxHidden) +
                   ", 1 <= A <= " + std::to_string(kPolicyMaxActions) + ", O >= 1)");
    return R2D2_ERR_UNSUPPORTED;
  }
  ExploreArgs e = {};
  if (explore) {
    const bool ou = explore->kind == R2D2_EXPLORATION_OU;
    R2D2_REQUIRE(ou || explore->kind == R2D2_EXPLORATION_GAUSSIAN,
                 "kind is R2D2_EXPLORATION_GAUSSIAN or R2D2_EXPLORATION_OU");
    R2D2_REQUIRE(explore->actor_id && explore->sigma && action, "null");
    R2D2_REQUIRE(ou == (explore->ou_state != nullptr), "ou_state is given under OU and NULL under GAUSSIAN");
    R2D2_REQUIRE(!ou || (explore->one_minus_theta >= 0.0f && explore->one_minus_theta < 1.0f),
                 "one_minus_theta = 1 - theta with theta in (0, 1]");
    const size_t NA = (size_t)N * A;
    R2D2_REQUIRE(action + NA <= mu || mu + NA <= action, "action must not overlap mu");
    std::vector<float> sigma(N);
    R2D2_CUDA_TRY(cudaMemcpyAsync(sigma.data(), explore->sigma, sizeof(float) * N, cudaMemcpyDeviceToHost, stream));
    R2D2_CUDA_TRY(cudaStreamSynchronize(stream));
    for (int n = 0; n < N; ++n)
      if (!(sigma[n] >= 0.0f && std::isfinite(sigma[n]))) {
        set_last_error("r2d2_policy_step_explore: sigma[" + std::to_string(n) + "] = " + std::to_string(sigma[n]) +
                       " (allowed: finite and >= 0)");
        return R2D2_ERR_ARG;
      }
    e.actor_id = explore->actor_id; e.sigma = explore->sigma; e.ou_state = explore->ou_state; e.action = action;
    e.seed = explore->seed; e.step_lo = (uint32_t)explore->step; e.step_hi = (uint32_t)(explore->step >> 32);
    e.one_minus_theta = explore->one_minus_theta;
  }
  StepArgs a;
  a.p0 = params[0]; a.p1 = params[1]; a.p2 = params[2]; a.p3 = params[3];
  a.obs = obs; a.state_in = state_in; a.state_out = state_out; a.mu = mu;
  a.G = workspace;
  a.Z = a.G + (size_t)N * H * 16;
  a.mu_t = a.Z + (size_t)N * H * 4;
  a.N = N; a.O = O; a.A = A; a.H = H;
  a.obs_mean = obs_mean; a.obs_inv_std = obs_inv_std; a.obs_clip = obs_clip;
  const unsigned tiles = (unsigned)ceil_div(N, NT);
  const unsigned head_blocks = (unsigned)ceil_div(ceil_div(A, 4), WARPS);
  const dim3 grid1(H / WARPS + H / (4 * WARPS), tiles, 4);
  if (obs_mean) R2D2_TRY(launch_phase(policy_obs_norm_phase1_kernel, grid1, a, stream));
  else R2D2_TRY(launch_phase(policy_phase_kernel<1>, grid1, a, stream));
  R2D2_TRY(launch_phase(policy_phase_kernel<2>, dim3(H / WARPS, tiles, 2), a, stream));
  const dim3 grid3(head_blocks, tiles, 2);
  if (!explore) R2D2_TRY(launch_phase(policy_phase_kernel<3>, grid3, a, stream));
  else if (explore->kind == R2D2_EXPLORATION_OU)
    R2D2_TRY(launch_phase(policy_explore_head_kernel<kOU>, grid3, a, stream, e));
  else
    R2D2_TRY(launch_phase(policy_explore_head_kernel<kGaussian>, grid3, a, stream, e));
  R2D2_TRY(launch_phase(policy_phase_kernel<4>, dim3(H / (4 * WARPS), tiles, 2), a, stream));
  R2D2_TRY(launch_phase(policy_phase_kernel<5>, dim3(H / WARPS, tiles, 2), a, stream));
  return R2D2_OK;
}

}  // namespace r2d2

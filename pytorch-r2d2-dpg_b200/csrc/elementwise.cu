// HBM-bound pieces of the learner path: fused n-step target / value rescaling / TD loss gradient /
// sequence priority (learner.py:107-111,135-138; utils.py:17-21), Adam (learner.py:50-53,114,128),
// bias-gradient column sums, small reductions.
#include "elementwise.cuh"

#include <cmath>
#include <map>
#include <mutex>
#include <utility>

namespace r2d2 {
namespace {

__device__ __forceinline__ float value_rescale(float x) {
  // h(x) = sign(x) * (sqrt(|x| + 1) - 1), utils.py:20-21 (no eps*x term, no inverse anywhere)
  const float m = sqrtf(fabsf(x) + 1.0f) - 1.0f;
  return x > 0.f ? m : (x < 0.f ? -m : 0.f);
}

// ---- R2D2's invertible value rescaling (TdPriorityParams::rescaling = R2D2_RESCALE_INVERTIBLE), in forms that stay
// accurate in fp32 near zero, where critic outputs start (l3 ~ U(+-3e-3)); the textbook closed forms cancel there.
// h_eps(x) = sign(x) (sqrt(|x| + 1) - 1) + eps x, with sqrt(a + 1) - 1 written as a / (sqrt(a + 1) + 1).
__device__ __forceinline__ float value_rescale_eps(float x, float eps) {
  const float a = fabsf(x);
  return copysignf(a / (sqrtf(a + 1.0f) + 1.0f), x) + eps * x;
}
// h_eps^-1(x) = sign(x) v (v + 2), v = sqrt(s + 1) - 1 the positive root of eps v^2 + (1 + 2 eps) v - |x| = 0, taken as
// 2 |x| / ((1 + 2 eps) + sqrt((1 + 2 eps)^2 + 4 eps |x|)): no step cancels, and eps = 0 gives v = |x|.
__device__ __forceinline__ float inverse_value_rescale(float x, float eps) {
  const float a = fabsf(x);
  const float c = 1.0f + 2.0f * eps;
  const float v = (2.0f * a) / (c + sqrtf(c * c + 4.0f * eps * a));
  return copysignf(v * (v + 2.0f), x);
}

// the n-step target of one element: reference h0(r + cont q'), or invertible h_eps(r + cont h_eps^-1(q'))
template <bool kInvertible>
__device__ __forceinline__ float td_target(float r, float cont, float qn, float eps) {
  if (kInvertible) return value_rescale_eps(r + cont * inverse_value_rescale(qn, eps), eps);
  return value_rescale(r + cont * qn);
}

// what a time step contributes to its sequence's priority: the squared TD (reference) or its root, the RMS over actions
template <bool kAbs>
__device__ __forceinline__ float priority_term(float td_sq) { return kAbs ? sqrtf(td_sq) : td_sq; }

// fallback (no td_sq buffer to reduce through): grid ceil(B/32) CTAs, 1024 threads = 32 warps; lane -> batch column, warp -> time rows i = w, w+32, ...
// (the kernel moves ~1 MB: it is bound by the length of the per-thread dependent load chain, hence the wide block)
// <false, false> is the reference's target and squared-error priority; see td_target / priority_term for the others.
constexpr int TD_WARPS = 32;
template <bool kInvertible, bool kAbs>
__global__ void __launch_bounds__(TD_WARPS * 32) td_priority_column_kernel(TdPriorityParams p, float* loss_part) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int b = blockIdx.x * 32 + lane;
  const int L = p.L, B = p.B, A = p.A;
  const float inv_a = 1.0f / (float)A;
  const float grad_scale = 2.0f / ((float)L * (float)B * (float)A);
  float run_max = -INFINITY, run_sum = 0.f, sq_total = 0.f;
  if (b < B) {
    // importance weight of sequence b: scales its share of the loss and of dq; td_sq and the priority stay unweighted
    const float wb = p.is_weight ? __ldg(p.is_weight + b) : 1.0f;
    const float gs = grad_scale * wb;
    for (int i = w; i < L; i += TD_WARPS) {
      const float r = __ldg(p.rew + (size_t)(p.burn_in + i) * B + b);
      const float d = __ldg(p.term + (size_t)(p.burn_in + i + p.n_step - 1) * B + b);
      const float cont = p.gamma_n * (1.0f - d);
      const size_t base = ((size_t)i * B + b) * A;
      float sq = 0.f;
      for (int a = 0; a < A; ++a) {
        const float q = __ldg(p.q + base + a);
        const float y = td_target<kInvertible>(r, cont, __ldg(p.q_next + base + a), p.eps);
        const float diff = q - y;
        if (p.target) p.target[base + a] = y;
        if (p.dq) p.dq[base + a] = gs * diff;
        sq += diff * diff;
      }
      sq_total += wb * sq;
      const float td = sq * inv_a;
      if (p.td_sq) p.td_sq[(size_t)i * B + b] = td;
      // learner.py:137 `average_td_loss[b:-1:B]` drops flat index L*B-1, i.e. (i=L-1, b=B-1)
      if (!(i == L - 1 && b == B - 1)) {
        const float m = priority_term<kAbs>(td);
        run_max = fmaxf(run_max, m);
        run_sum += m;
      }
    }
  }
  __shared__ float s_max[TD_WARPS][32], s_sum[TD_WARPS][32], s_sq[TD_WARPS];
  s_max[w][lane] = run_max;
  s_sum[w][lane] = run_sum;
  const float wsq = warp_sum(sq_total);
  if (lane == 0) s_sq[w] = wsq;
  __syncthreads();
  if (w == 0) {
    float mx = s_max[0][lane], sm = s_sum[0][lane];
#pragma unroll
    for (int k = 1; k < TD_WARPS; ++k) { mx = fmaxf(mx, s_max[k][lane]); sm += s_sum[k][lane]; }
    if (b < B && p.priority) {
      const int count = L - ((b == B - 1) ? 1 : 0);
      p.priority[b] = p.eta * mx + (1.0f - p.eta) * (sm / (float)count);  // utils.py:17-18
    }
    if (lane == 0 && loss_part) {
      float tot = 0.f;
#pragma unroll
      for (int k = 0; k < TD_WARPS; ++k) tot += s_sq[k];
      loss_part[blockIdx.x] = tot / ((float)L * (float)B * (float)A);
    }
  }
}

// ---- the path's TD kernel pair (learner.py:107-111,135-138): every global access is a lane-contiguous 128-byte line.
// Pass 1, one warp per (time row i, 32 consecutive batch elements): the [32 x A] spans of q and q_next are ONE contiguous
// run of 32*A floats each (layout [L][B][A]); the warp copies them into shared memory with unit-stride loads, every lane
// then owns one batch element (A values, stride-A shared reads: conflict free for odd A, 2-way for A = 6), writes the
// target and the loss gradient back into the same shared slots and the warp stores them with unit-stride writes.
// Pass 2 reduces td_sq[L,B] per batch element (max / mean with the [b:-1:B] quirk) and sums the loss: lanes along b.
constexpr int TD1_WARPS = 8;
template <bool kInvertible>
__global__ void __launch_bounds__(TD1_WARPS * 32) td_elem_kernel(TdPriorityParams p) {
  extern __shared__ float td_smem[];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int L = p.L, B = p.B, A = p.A;
  const int i = blockIdx.y * TD1_WARPS + w;
  const int b0 = blockIdx.x * 32;
  if (i >= L) return;
  const int nb = min(32, B - b0), span = nb * A;
  float* sq_ = td_smem + (size_t)w * 2 * 32 * A;       // q, then (in place) dq
  float* sn_ = sq_ + 32 * A;                           // q_next, then (in place) target
  const size_t base = ((size_t)i * B + b0) * A;
  for (int k = lane; k < span; k += 32) {
    sq_[k] = __ldg(p.q + base + k);
    sn_[k] = __ldg(p.q_next + base + k);
  }
  __syncwarp();
  const float grad_scale = 2.0f / ((float)L * (float)B * (float)A);
  if (lane < nb) {
    const int b = b0 + lane;
    const float r = __ldg(p.rew + (size_t)(p.burn_in + i) * B + b);
    const float d = __ldg(p.term + (size_t)(p.burn_in + i + p.n_step - 1) * B + b);
    const float cont = p.gamma_n * (1.0f - d);
    const float gs = grad_scale * (p.is_weight ? __ldg(p.is_weight + b) : 1.0f);   // w = 1: exactly grad_scale
    float sq = 0.f;
    for (int a = 0; a < A; ++a) {
      const float y = td_target<kInvertible>(r, cont, sn_[lane * A + a], p.eps);
      const float diff = sq_[lane * A + a] - y;
      sn_[lane * A + a] = y;
      sq_[lane * A + a] = gs * diff;
      sq += diff * diff;
    }
    p.td_sq[(size_t)i * B + b] = sq / (float)A;
  }
  __syncwarp();
  if (p.target) for (int k = lane; k < span; k += 32) p.target[base + k] = sn_[k];
  if (p.dq) for (int k = lane; k < span; k += 32) p.dq[base + k] = sq_[k];
}

constexpr int TD2_WARPS = 8;
template <bool kAbs>
__global__ void __launch_bounds__(TD2_WARPS * 32) td_reduce_kernel(TdPriorityParams p, float* loss_part) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int b = blockIdx.x * 32 + lane;
  const int L = p.L, B = p.B;
  float run_max = -INFINITY, run_sum = 0.f, tot = 0.f;
  if (b < B) {
    const float wb = p.is_weight ? __ldg(p.is_weight + b) : 1.0f;   // w = 1: w * td + tot rounds like td + tot
    for (int i = w; i < L; i += TD2_WARPS) {
      const float td = p.td_sq[(size_t)i * B + b];
      tot += wb * td;
      // learner.py:137 `average_td_loss[b:-1:B]` drops flat index L*B-1, i.e. (i=L-1, b=B-1)
      if (!(i == L - 1 && b == B - 1)) {
        const float m = priority_term<kAbs>(td);
        run_max = fmaxf(run_max, m);
        run_sum += m;
      }
    }
  }
  __shared__ float s_max[TD2_WARPS][32], s_sum[TD2_WARPS][32], s_tot[TD2_WARPS][32];
  s_max[w][lane] = run_max; s_sum[w][lane] = run_sum; s_tot[w][lane] = tot;
  __syncthreads();
  if (w == 0) {
    float mx = s_max[0][lane], sm = s_sum[0][lane], tt = s_tot[0][lane];
#pragma unroll
    for (int k = 1; k < TD2_WARPS; ++k) { mx = fmaxf(mx, s_max[k][lane]); sm += s_sum[k][lane]; tt += s_tot[k][lane]; }
    if (b < B && p.priority) {
      const int count = L - ((b == B - 1) ? 1 : 0);
      p.priority[b] = p.eta * mx + (1.0f - p.eta) * (sm / (float)count);  // utils.py:17-18
    }
    tt = warp_sum(tt);   // critic loss = mean over (i, b, a) of w_b diff^2 = sum of w_b td_sq / (L * B)
    if (lane == 0 && loss_part) loss_part[blockIdx.x] = tt / ((float)L * (float)B);
  }
}

__global__ void __launch_bounds__(256) colsum_kernel(const float* __restrict__ x, long long ld, int M, int N,
                                                     int rows_per_block, float* __restrict__ part) {
  // block = 32 columns x 8 row lanes; grid.x over column chunks, grid.y over row ranges; row range y writes slice y
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int col = blockIdx.x * 32 + lane;
  const int r0 = blockIdx.y * rows_per_block;
  const int r1 = min(M, r0 + rows_per_block);
  float acc = 0.f;
  if (col < N)
    for (int r = r0 + w; r < r1; r += 8) acc += __ldg(x + (size_t)r * ld + col);
  __shared__ float sm[8][32];
  sm[w][lane] = acc;
  __syncthreads();
  if (w == 0 && col < N) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += sm[k][lane];
    part[(size_t)blockIdx.y * N + col] = t;
  }
}

// kClip: the gradient is multiplied by the clip coefficient grad_norm_kernel left at *clip_coef (one load per thread).
// kPolyak: the target net is blended with the post-step weight while it is still in a register,
// target = fl(fl(target * tau_keep) + fl(param' * tau)) - two rounded products and one rounded add, as utils.soft_update
// computes it with torch.  <false, false> is the plain optimiser step; its extra arguments are never read.
template <bool kClip, bool kPolyak>
__global__ void __launch_bounds__(256) adam_kernel(float* __restrict__ param, const float* __restrict__ grad,
                                                   float* __restrict__ m, float* __restrict__ v, long long n,
                                                   float grad_scale, float beta1, float beta2, float step_size,
                                                   float inv_bc2_sqrt, float eps, const float* __restrict__ clip_coef,
                                                   float* __restrict__ target, float tau_keep, float tau) {
  const float c = kClip ? *clip_coef : 1.0f;
  // torch.optim.Adam single-tensor math (learner.py:50,52 defaults): lerp m, addcmul v, sqrt/bc2 + eps, addcdiv
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float g = grad[i] * grad_scale;
    if (kClip) g = __fmul_rn(g, c);   // c = 1: the unclipped bits
    const float mi = m[i] + (g - m[i]) * (1.0f - beta1);
    // the fused variants spell out the contraction the plain kernel compiles v's update to, fma(v, b2, ((1 - b2) g) g):
    // left to itself the compiler contracts it as fma(g, (1 - b2) g, v b2) there, and c = 1 would change the bits
    const float vi = (kClip || kPolyak) ? __fmaf_rn(v[i], beta2, __fmul_rn(__fmul_rn(1.0f - beta2, g), g))
                                        : v[i] * beta2 + (1.0f - beta2) * g * g;
    m[i] = mi;
    v[i] = vi;
    const float denom = sqrtf(vi) * inv_bc2_sqrt + eps;
    const float p = param[i] - step_size * (mi / denom);
    param[i] = p;
    if (kPolyak) target[i] = __fadd_rn(__fmul_rn(target[i], tau_keep), __fmul_rn(p, tau));
  }
}

// Global L2 norm of grad * grad_scale (torch.nn.utils.clip_grad_norm_ over one net's flat block) and the clip
// coefficient, without a host round trip and without floating-point atomics: a fixed grid of kGradNormBlocks CTAs writes
// one partial sum of squares each; the CTA that draws the last ticket adds the partials in a fixed order, writes
// norm = N, coef = min(1, max_norm / (N + 1e-6)) and resets the ticket for the next launch.  Same inputs, same bits.
// Squares are summed in double: a float times a float is exact there, so N is well within 1e-6 of float64.
constexpr int NORM_THREADS = 256;

__device__ __forceinline__ double block_sum_f64(double x, double* s) {   // result valid in thread 0
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = x;
  __syncthreads();
  double t = 0.0;
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < NORM_THREADS / 32; ++k) t += s[k];
  }
  return t;
}

__global__ void __launch_bounds__(NORM_THREADS) grad_norm_kernel(const float* __restrict__ grad, long long n,
                                                                 float grad_scale, float max_norm, double* part,
                                                                 unsigned int* ticket, float* __restrict__ norm,
                                                                 float* __restrict__ coef) {
  __shared__ double s_part[NORM_THREADS / 32];
  __shared__ double s_last[NORM_THREADS / 32];
  __shared__ bool last;
  double acc = 0.0;
  for (long long i = blockIdx.x * (long long)NORM_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * NORM_THREADS) {
    const float g = grad[i] * grad_scale;   // the gradient exactly as adam_kernel forms it
    acc += (double)g * (double)g;
  }
  acc = block_sum_f64(acc, s_part);
  if (threadIdx.x == 0) {
    part[blockIdx.x] = acc;
    __threadfence();                        // the partial is visible device-wide before the ticket is drawn
    last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  double t = 0.0;
  for (int k = threadIdx.x; k < (int)gridDim.x; k += NORM_THREADS) t += __ldcg(part + k);
  t = block_sum_f64(t, s_last);
  if (threadIdx.x == 0) {
    const float nrm = (float)sqrt(t);
    *norm = nrm;
    *coef = fminf(1.0f, max_norm / (nrm + 1e-6f));
    *ticket = 0u;
  }
}

__global__ void __launch_bounds__(256) fill_kernel(float* __restrict__ x, long long n, float value) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    x[i] = value;
}

__global__ void __launch_bounds__(256) scaled_sum_kernel(const float* __restrict__ x, long long n, float scale,
                                                         float* __restrict__ part) {
  float acc = 0.f;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    acc += x[i];
  acc = warp_sum(acc);
  __shared__ float sm[8];
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int k = 0; k < 8; ++k) t += sm[k];
    part[blockIdx.x] = t * scale;
  }
}

__global__ void __launch_bounds__(256) add_partials_kernel(const float* __restrict__ part, int slices, int rows, int cols,
                                                           float* __restrict__ dst, long long ld_dst, float* __restrict__ dst2) {
  const long long n = (long long)rows * cols, stride = n;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float t = 0.f;
    for (int s = 0; s < slices; ++s) t += part[s * stride + i];
    const long long r = i / cols, c = i % cols;
    dst[r * ld_dst + c] += t;
    if (dst2) dst2[r * ld_dst + c] += t;
  }
}

__global__ void add_vec_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = a[i] + b[i];
}

__global__ void mul_dtanh_kernel(const float* __restrict__ d_out, const float* __restrict__ out,
                                 float* __restrict__ d_pre, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    d_pre[i] = d_out[i] * (1.0f - out[i] * out[i]);
}

// ---- actor-side next rows (SURVEY 8f N2): n-step reward pre-sum (actor.py:74-76) and the initial priorities of a
// finished episode (actor.py:78-107), batched over episodes (time-major [T,B], one episode per batch column, zero
// padded past its last row).
__global__ void __launch_bounds__(256) nstep_reward_kernel(const float* __restrict__ raw, const int* __restrict__ n_rows,
                                                           int T, int B, int n_step, float gamma, float* __restrict__ out) {
  const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= (long long)T * B) return;
  const int i = (int)(idx / B), b = (int)(idx % B);
  float v = raw[idx];
  if (i < n_rows[b] - n_step) {   // rows of the real episode: discounted sum of the next n raw rewards
    double acc = 0.0, g = 1.0;
    for (int j = 0; j < n_step; ++j) { acc += (double)raw[(size_t)(i + j) * B + b] * g; g *= (double)gamma; }
    v = (float)acc;
  }
  out[idx] = v;
}

// priority k of episode b: 0.9 max + 0.1 mean over j = k+Bn+1 .. k+Bn+L of td_j^2,
// td_j = mean_A(q[j,b,:] - h(R[j,b] + gamma^n (1 - term[j+n-1,b]) q_next[j+n,b,:]))  -  the reference's deque of
// `learning` entries is one step ahead of the window the learner trains on (actor.py:102-107), reproduced here.
// kInvertible: the target of td_target<true>.  kAbs: |td_j| in place of td_j^2 - still the MEAN difference over actions,
// where the learner's abs metric takes the RMS; the two sides differ here as they do in the squared metric.
template <bool kInvertible, bool kAbs>
__global__ void __launch_bounds__(128) actor_priority_kernel(const float* __restrict__ q, const float* __restrict__ q_next,
                                                             const float* __restrict__ rew, const float* __restrict__ term,
                                                             const int* __restrict__ n_rows, int B, int A, int burn_in,
                                                             int learning, int n_step, float gamma_n, float eta,
                                                             int p_max, float* __restrict__ prio, float eps) {
  const int b = blockIdx.y;
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= p_max) return;
  const int E = n_rows[b] - n_step;
  float out = 0.f;
  int k_out = k;
  if (k < E - (burn_in + learning)) {
    float mx = -INFINITY, sum = 0.f;
    int j = k + burn_in + 1;
    for (; j <= k + burn_in + learning; ++j) {
      const float r = rew[(size_t)j * B + b];
      const float cont = gamma_n * (1.0f - term[(size_t)(j + n_step - 1) * B + b]);
      const float* qj = q + ((size_t)j * B + b) * A;
      const float* qn = q_next + ((size_t)(j + n_step) * B + b) * A;
      float acc = 0.f;
      if (kInvertible) {   // one element at a time: unrolled, its two divisions' slow paths would keep more live
#pragma unroll 1
        for (int a = 0; a < A; ++a) acc += qj[a] - td_target<true>(r, cont, qn[a], eps);
      } else {
        for (int a = 0; a < A; ++a) acc += qj[a] - td_target<false>(r, cont, qn[a], eps);
      }
      const float td = acc / (float)A;
      const float sq = kAbs ? fabsf(td) : td * td;
      mx = fmaxf(mx, sq);
      sum += sq;
    }
    out = eta * mx + (1.0f - eta) * (sum / (float)learning);
    // the new variants take k back from the loop counter: k itself, kept across the division slow-path calls of the
    // loop, costs the default variant 8 bytes of stack (its code stays as it was)
    if (kInvertible || kAbs) k_out = j - (burn_in + learning + 1);
  }
  prio[(size_t)b * p_max + k_out] = out;
}

}  // namespace

int nstep_rewards(const float* raw, const int* n_rows, int T, int B, int n_step, float gamma, float* out, cudaStream_t stream) {
  R2D2_REQUIRE(raw && n_rows && out && raw != out && T > 0 && B > 0 && n_step > 0, "nstep_rewards args");
  nstep_reward_kernel<<<(unsigned)(((long long)T * B + 255) / 256), 256, 0, stream>>>(raw, n_rows, T, B, n_step, gamma, out);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

int actor_priorities(const float* q, const float* q_next, const float* rew, const float* term, const int* n_rows, int B,
                     int A, int burn_in, int learning, int n_step, float gamma, float eta, int p_max, float* prio,
                     cudaStream_t stream, const TdOptions& opt) {
  R2D2_REQUIRE(q && q_next && rew && term && n_rows && prio && B > 0 && A > 0 && p_max > 0, "actor_priorities args");
  R2D2_TRY(check_td_options(opt));
  const float gamma_n = (float)std::pow((double)gamma, (double)n_step);
  const bool inv = opt.rescaling == kRescaleInvertible, abs_ = opt.priority_metric == kPriorityAbs;
  auto kernel = inv ? (abs_ ? actor_priority_kernel<true, true> : actor_priority_kernel<true, false>)
                    : (abs_ ? actor_priority_kernel<false, true> : actor_priority_kernel<false, false>);
  kernel<<<dim3(ceil_div(p_max, 128), B), 128, 0, stream>>>(q, q_next, rew, term, n_rows, B, A, burn_in, learning, n_step,
                                                           gamma_n, eta, p_max, prio, opt.eps);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

int add_vec(const float* a, const float* b, float* out, int n, cudaStream_t stream) {
  add_vec_kernel<<<ceil_div(n, 256), 256, 0, stream>>>(a, b, out, n);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

int mul_dtanh(const float* d_out, const float* out, float* d_pre, long long n, cudaStream_t stream) {
  int blocks = (int)((n + 255) / 256);
  if (blocks > num_sms() * 8) blocks = num_sms() * 8;
  mul_dtanh_kernel<<<blocks, 256, 0, stream>>>(d_out, out, d_pre, n);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

int check_td_options(const TdOptions& opt) {
  R2D2_REQUIRE(opt.rescaling == kRescaleReference || opt.rescaling == kRescaleInvertible,
               "value rescaling is R2D2_RESCALE_REFERENCE (0) or R2D2_RESCALE_INVERTIBLE (1)");
  R2D2_REQUIRE(opt.priority_metric == kPrioritySquared || opt.priority_metric == kPriorityAbs,
               "priority metric is R2D2_PRIORITY_SQUARED (0) or R2D2_PRIORITY_ABS (1)");
  R2D2_REQUIRE(opt.rescaling == kRescaleReference || (opt.eps >= 0.0f && opt.eps <= 1.0f),
               "rescaling eps lies in [0, 1]");   // NaN fails both comparisons
  return R2D2_OK;
}

int td_priority(const TdPriorityParams& params, cudaStream_t stream, const TdOptions& opt) {
  R2D2_REQUIRE(params.q && params.q_next && params.rew && params.term, "null input");
  R2D2_REQUIRE(params.L > 0 && params.B > 0 && params.A > 0, "shape");
  R2D2_REQUIRE(!params.priority || params.L >= 2, "a priority output needs L >= 2: the [b:-1:B] series of the last "
                                                  "batch element drops its last TD step, so L = 1 leaves it empty");
  R2D2_TRY(check_td_options(opt));
  const bool inv = opt.rescaling == kRescaleInvertible, abs_ = opt.priority_metric == kPriorityAbs;
  TdPriorityParams p = params;
  p.eps = opt.eps;
  const int col_blocks = ceil_div(p.B, 32);
  float* loss_part = nullptr;     // one partial loss per column block, summed in block order
  if (p.loss_sum) {
    R2D2_CUDA_TRY(cudaMemsetAsync(p.loss_sum, 0, sizeof(float), stream));
    R2D2_TRY(partials_scratch(col_blocks, stream, &loss_part));
  }
  const size_t smem = (size_t)TD1_WARPS * 2 * 32 * p.A * sizeof(float);
  if (p.td_sq && smem <= 48 * 1024) {   // the path's configuration: two line-coalesced passes over L x B x A and L x B
    auto elem = inv ? td_elem_kernel<true> : td_elem_kernel<false>;
    elem<<<dim3(col_blocks, ceil_div(p.L, TD1_WARPS)), TD1_WARPS * 32, smem, stream>>>(p);
    count_launch();
    if (p.priority || p.loss_sum) {
      auto reduce = abs_ ? td_reduce_kernel<true> : td_reduce_kernel<false>;
      reduce<<<col_blocks, TD2_WARPS * 32, 0, stream>>>(p, loss_part);
      count_launch();
    }
  } else {
    auto column = inv ? (abs_ ? td_priority_column_kernel<true, true> : td_priority_column_kernel<true, false>)
                      : (abs_ ? td_priority_column_kernel<false, true> : td_priority_column_kernel<false, false>);
    column<<<col_blocks, TD_WARPS * 32, 0, stream>>>(p, loss_part);
    count_launch();
  }
  R2D2_CUDA_TRY(cudaGetLastError());
  if (p.loss_sum) R2D2_TRY(add_partials(loss_part, col_blocks, 1, 1, p.loss_sum, 1, nullptr, stream));
  return R2D2_OK;
}

int colsum(const float* x, long long ld, int M, int N, float* out, float* out2, cudaStream_t stream) {
  R2D2_REQUIRE(x && out && M > 0 && N > 0, "colsum args");
  const int col_blocks = ceil_div(N, 32);
  int row_blocks = ceil_div(4 * num_sms(), col_blocks);
  if (row_blocks > ceil_div(M, 64)) row_blocks = ceil_div(M, 64);
  if (row_blocks < 1) row_blocks = 1;
  const int rows_per_block = ceil_div(M, row_blocks);
  const int slices = ceil_div(M, rows_per_block);
  float* part = nullptr;
  R2D2_TRY(partials_scratch((size_t)slices * N, stream, &part));
  colsum_kernel<<<dim3(col_blocks, slices), 256, 0, stream>>>(x, ld, M, N, rows_per_block, part);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return add_partials(part, slices, 1, N, out, N, out2, stream);
}

int adam_step(float* param, const float* grad, float* m, float* v, long long n, int step, float lr, float beta1,
              float beta2, float eps, float grad_scale, cudaStream_t stream, const float* clip_coef, float* target,
              float tau) {
  R2D2_REQUIRE(param && grad && m && v && n > 0 && step >= 1, "adam args");
  R2D2_REQUIRE(!target || (tau > 0.0f && tau <= 1.0f), "Polyak weight");
  const double bc1 = 1.0 - pow((double)beta1, (double)step);
  const double bc2 = 1.0 - pow((double)beta2, (double)step);
  const float step_size = (float)((double)lr / bc1);
  const float inv_bc2_sqrt = (float)(1.0 / sqrt(bc2));
  const float tau_keep = (float)(1.0 - (double)tau);   // how torch rounds the Python scalar (1.0 - tau)
  int blocks = (int)((n + 255) / 256);
  if (blocks > num_sms() * 8) blocks = num_sms() * 8;
  auto kernel = clip_coef ? (target ? adam_kernel<true, true> : adam_kernel<true, false>)
                          : (target ? adam_kernel<false, true> : adam_kernel<false, false>);
  kernel<<<blocks, 256, 0, stream>>>(param, grad, m, v, n, grad_scale, beta1, beta2, step_size, inv_bc2_sqrt, eps,
                                     clip_coef, target, tau_keep, tau);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

int grad_norm(const float* grad, long long n, float grad_scale, float max_norm, double* partials, unsigned int* ticket,
              float* norm, float* coef, cudaStream_t stream) {
  R2D2_REQUIRE(grad && partials && ticket && norm && coef && n > 0 && max_norm >= 0.0f, "grad_norm args");
  grad_norm_kernel<<<kGradNormBlocks, NORM_THREADS, 0, stream>>>(grad, n, grad_scale, max_norm, partials, ticket, norm,
                                                                coef);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

int fill_f32(float* x, long long n, float value, cudaStream_t stream) {
  int blocks = (int)((n + 255) / 256);
  if (blocks > num_sms() * 8) blocks = num_sms() * 8;
  fill_kernel<<<blocks, 256, 0, stream>>>(x, n, value);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

int scaled_sum(const float* x, long long n, float scale, float* out, cudaStream_t stream) {
  R2D2_CUDA_TRY(cudaMemsetAsync(out, 0, sizeof(float), stream));
  int blocks = (int)((n + 255) / 256);
  if (blocks > num_sms() * 4) blocks = num_sms() * 4;
  float* part = nullptr;
  R2D2_TRY(partials_scratch(blocks, stream, &part));
  scaled_sum_kernel<<<blocks, 256, 0, stream>>>(x, n, scale, part);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return add_partials(part, blocks, 1, 1, out, 1, nullptr, stream);
}

namespace {
struct PartialsBuf { float* ptr = nullptr; size_t floats = 0; };
std::mutex g_partials_mutex;
std::map<std::pair<int, cudaStream_t>, PartialsBuf> g_partials;
}  // namespace

int partials_scratch(size_t floats, cudaStream_t stream, float** out) {
  int dev = 0;
  R2D2_CUDA_TRY(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(g_partials_mutex);
  PartialsBuf& b = g_partials[std::make_pair(dev, stream)];
  if (b.floats < floats) {
    if (b.ptr) { R2D2_CUDA_TRY(cudaDeviceSynchronize()); R2D2_CUDA_TRY(cudaFree(b.ptr)); b.ptr = nullptr; b.floats = 0; }
    const size_t want = floats + floats / 4 + (1u << 16);
    R2D2_CUDA_TRY(cudaMalloc(&b.ptr, want * sizeof(float)));
    b.floats = want;
  }
  *out = b.ptr;
  return R2D2_OK;
}

int add_partials(const float* part, int slices, int rows, int cols, float* dst, long long ld_dst, float* dst2,
                 cudaStream_t stream) {
  R2D2_REQUIRE(part && dst && slices >= 1 && rows >= 1 && cols >= 1 && ld_dst >= cols, "add_partials args");
  const long long n = (long long)rows * cols;
  int blocks = (int)((n + 255) / 256);
  if (blocks > num_sms() * 8) blocks = num_sms() * 8;
  add_partials_kernel<<<blocks, 256, 0, stream>>>(part, slices, rows, cols, dst, ld_dst, dst2);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

}  // namespace r2d2

// GPU-resident prioritized sequence replay shard (replaces LearnerReplayMemory, replay_memory.py:67-175).
//
// HBM layout (SoA, one "row" per stored env step incl. the n_step pad rows of actor.py:173):
//   obs_rows [cap,O]  act_rows [cap,A]  rew_rows [cap]  term_rows [cap]  state_rows [cap,4,2,H]
// state_rows is fp32, or fp16 under R2D2_STATE_F16 (rounded once at ingest, widened back to fp32 by the gather); under
// R2D2_STATE_MEMORY_HOST it lives in mapped, page-locked host memory and everything else stays in HBM.  Ingest and
// restore write state rows through one path for both types and both tiers: stage_states decides whether the call's
// states go through the device staging block, store_states writes a run of ring rows from wherever they are (a copy,
// or a rounding / widening kernel), and write_rows puts a run's obs / act / rew / term next to them.
// Episodes occupy contiguous row ranges of a ring; FIFO eviction (replay_memory.py:148-152).
// Sum tree: one leaf per ROW (priority 0 for rows that are not valid sequence starts), fan-out 32:
// every node is the left-to-right fp32 sum of its 32 children (one 128-byte line), so the tree has
// ceil(log32(cap)) levels (5 for 2M rows) instead of 21 dependent loads of a binary tree, and the
// CUDA tree and its C restatement (oracle/sumtree_oracle.c) are bit-identical by construction.
#include <cuda_fp16.h>
#include <float.h>

#include <algorithm>
#include <cstring>
#include <deque>
#include <map>
#include <vector>

#include "obs_norm.cuh"
#include "peer_sync.cuh"
#include "replay.cuh"

namespace r2d2 {

namespace {

// Descent from the root with residual r: the leaf index, and in *v (kLeafValue) the drawn leaf's value.
template <bool kLeafValue>
__device__ __forceinline__ long long tree_descend(const TreeView& tv, float r, float* leaf_val) {
  const int top = tv.levels - 1;
  long long idx = 0;
  float v = 0.f;   // value of the picked child; after the level-1 pass that is the leaf itself
  for (int l = top; l >= 1; --l) {
    const float4* ch4 = reinterpret_cast<const float4*>(tv.lvl[l - 1] + idx * TREE_K);
    float c[TREE_K];
#pragma unroll
    for (int k = 0; k < TREE_K / 4; ++k) {
      const float4 v4 = ch4[k];
      c[4 * k] = v4.x; c[4 * k + 1] = v4.y; c[4 * k + 2] = v4.z; c[4 * k + 3] = v4.w;
    }
    int pick = -1;
#pragma unroll
    for (int k = 0; k < TREE_K; ++k) {
      if (pick < 0) {
        if (r < c[k]) { pick = k; if (kLeafValue) v = c[k]; }
        else r = __fsub_rn(r, c[k]);
      }
    }
    if (pick < 0) {  // rounding pushed the residual past the last child: take the last non-empty child
      float cl = 0.f;
#pragma unroll
      for (int k = 0; k < TREE_K; ++k)
        if (c[k] > 0.f) { pick = k; cl = c[k]; }
      if (pick < 0) pick = 0;
      r = __fmul_rn(cl, 0.99999994f);
      if (kLeafValue) v = cl;
    }
    idx = idx * TREE_K + pick;
  }
  if (kLeafValue) *leaf_val = v;
  return idx;
}

// kLeafValue: also return the value of the drawn leaf (the weighted draw turns it into an importance weight)
template <bool kLeafValue>
__global__ void __launch_bounds__(256) tree_sample_kernel(TreeView tv, const float* __restrict__ u, int batch,
                                                          long long* __restrict__ leaf, float* __restrict__ leaf_val) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= batch) return;
  const float total = tv.lvl[tv.levels - 1][0];
  float v = 0.f;
  leaf[i] = tree_descend<kLeafValue>(tv, __fmul_rn(u[i], total), &v);
  if (kLeafValue) leaf_val[i] = v;
}

// Global draw (one CTA): the W shard roots are one more tree level above the shards, in rank order.  Every rank
// computes all W*B shard choices from the same totals and uniforms, so all ranks agree on the owner of every draw; the
// owner descends its own tree only for its draws, writes (leaf, shard, leaf value) into consumer j / B's fill slot,
// column j % B, and records the drawn leaf for the gather (-1 for the draws of other shards).  The walk over the roots
// is tree_descend's walk over 32 children, with one difference in the rounding fallback: it takes the last non-empty
// shard with the residual as it stood before that shard (the shard's own descent then clamps it), so that at W = 1 the
// residual reaching the shard is u * total unchanged - today's draw bit for bit.
template <bool kLeafValue>
__global__ void __launch_bounds__(1024) global_draw_kernel(TreeView tv, GlobalPeers p, GlobalLayout lay, int world,
                                                           int rank, int B, int slot, unsigned epoch) {
  __shared__ float s_min[32];
  char* own = p.base[rank];
  unsigned* flags = reinterpret_cast<unsigned*>(own);
  if ((int)threadIdx.x < world) spin_until(flags + kGlobalFlagTot + threadIdx.x, epoch, flags + kGlobalStatus);
  __syncthreads();
  const float* totals = reinterpret_cast<const float*>(own + kGlobalOffTotals);
  const float* u = reinterpret_cast<const float*>(own + lay.off_uniforms);
  long long* draw_leaf = reinterpret_cast<long long*>(own + lay.off_draw_leaf);
  float root[kGlobalMaxWorld];
  float total = 0.f;
  for (int k = 0; k < world; ++k) { root[k] = *reinterpret_cast<const volatile float*>(totals + k); total = __fadd_rn(total, root[k]); }
  float m = INFINITY;
  for (int j = threadIdx.x; j < world * B; j += blockDim.x) {
    const float r0 = __fmul_rn(*reinterpret_cast<const volatile float*>(u + j), total);
    float r = r0;
    int pick = -1;
    for (int k = 0; k < world; ++k) {
      if (pick < 0) {
        if (r < root[k]) pick = k;
        else r = __fsub_rn(r, root[k]);
      }
    }
    if (pick < 0) {   // rounding pushed the residual past the last root: the last non-empty shard, residual before it
      for (int k = 0; k < world; ++k)
        if (root[k] > 0.f) pick = k;
      if (pick < 0) pick = 0;
      r = r0;
      for (int k = 0; k < pick; ++k) r = __fsub_rn(r, root[k]);
    }
    if (pick != rank) { draw_leaf[j] = -1; continue; }
    float v = 0.f;
    const long long leaf = tree_descend<kLeafValue>(tv, r, &v);
    draw_leaf[j] = leaf;
    char* dst = p.base[j / B] + lay.slot(slot);
    reinterpret_cast<long long*>(dst + lay.off_leaf)[j % B] = leaf;
    reinterpret_cast<int*>(dst + lay.off_shard)[j % B] = rank;
    if (kLeafValue) {
      reinterpret_cast<float*>(dst + lay.off_weight)[j % B] = v;
      if (v > 0.f) m = fminf(m, v);
    }
  }
  if (kLeafValue) {   // the owner's minimum drawn leaf, sent with its delivery signal (global_deliver)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fminf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) s_min[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int k = 1; k < (int)(blockDim.x >> 5); ++k) m = fminf(m, s_min[k]);
      *reinterpret_cast<float*>(own + kGlobalOffOwnMin) = fminf(m, s_min[0]);
    }
  } else if (threadIdx.x == 0) {
    *reinterpret_cast<float*>(own + kGlobalOffOwnMin) = INFINITY;
  }
}

// Leaf stored for a priority p under the exponent alpha.  Zero stays zero (rows that start no sequence must stay
// undrawable, also at alpha = 0 where powf(0, 0) would be 1).
__device__ __forceinline__ float raise_priority(float p, float alpha) { return p > 0.f ? powf(p, alpha) : 0.f; }

__global__ void __launch_bounds__(256) raise_leaves_kernel(float* __restrict__ leaves, long long n, float alpha) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < n) leaves[i] = raise_priority(leaves[i], alpha);
}

// fp16 state storage, ingest.  A finite x with |x| >= 65520 (65504 + half an fp16 ulp) rounds to +-inf under
// round-to-nearest-even; NaN and +-inf are not counted (they pass through, as in fp32 storage).  Integer atomics, one
// per warp: the count does not depend on the schedule.
__global__ void __launch_bounds__(256) count_f16_overflow_kernel(const float* __restrict__ x, long long n,
                                                                 unsigned long long* __restrict__ count) {
  unsigned c = 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float a = fabsf(x[i]);
    c += (a >= 65520.f && a <= FLT_MAX) ? 1u : 0u;
  }
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(count, (unsigned long long)c);
}

// dst[i] = __float2half_rn(src[i]); n, src and dst are multiples of 8 elements (whole [4,2,H] rows: 8 H values), so
// every thread moves two float4 loads into one 16-byte store.
__global__ void __launch_bounds__(256) states_to_f16_kernel(const float* __restrict__ src, __half* __restrict__ dst,
                                                            long long n) {
  const long long n8 = n >> 3;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    const float4 a = reinterpret_cast<const float4*>(src)[2 * i];
    const float4 b = reinterpret_cast<const float4*>(src)[2 * i + 1];
    __half2 h[4] = {__floats2half2_rn(a.x, a.y), __floats2half2_rn(a.z, a.w), __floats2half2_rn(b.x, b.y),
                    __floats2half2_rn(b.z, b.w)};
    reinterpret_cast<uint4*>(dst)[i] = *reinterpret_cast<const uint4*>(h);
  }
}

// Exact fp16 -> fp32 widening of 4 halves (one 8-byte load) and of 8 halves (one 16-byte load)
__device__ __forceinline__ float4 widen4(uint2 v) {
  const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&v.x));
  const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&v.y));
  return make_float4(a.x, a.y, b.x, b.y);
}

struct Float8 { float4 lo, hi; };
__device__ __forceinline__ Float8 widen8(uint4 v) { return {widen4(make_uint2(v.x, v.y)), widen4(make_uint2(v.z, v.w))}; }

// fp16 states into an fp32 ring (snapshot restore of an fp16 file): dst[i] = (float)src[i], exact.  A stored range is
// whole [4,2,H] rows (8 H halves = 16 H bytes each, and the staging copy starts 16 bytes into its block), so both ends
// are 16-byte aligned for every H: each thread widens one 16-byte load of 8 halves into two float4 stores (the gather's
// widest route).
__global__ void __launch_bounds__(256) states_from_f16_kernel(const __half* __restrict__ src, float* __restrict__ dst,
                                                              long long n) {
  const long long n8 = n >> 3;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    const Float8 f = widen8(reinterpret_cast<const uint4*>(src)[i]);
    reinterpret_cast<float4*>(dst)[2 * i] = f.lo;
    reinterpret_cast<float4*>(dst)[2 * i + 1] = f.hi;
  }
}

// Snapshot restore: counts the imported leaves of one episode that no shard could have written - on its first n_valid
// rows (the sequence starts) a negative, NaN or infinite value, on the rows after them anything but zero.  Integer
// atomics, one per warp, as in count_f16_overflow_kernel.
__global__ void __launch_bounds__(256) count_bad_leaves_kernel(const float* __restrict__ leaves, long long n,
                                                               long long n_valid, unsigned long long* __restrict__ count) {
  unsigned c = 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float v = leaves[i];
    c += (i < n_valid ? !(v >= 0.f && v <= FLT_MAX) : v != 0.f) ? 1u : 0u;
  }
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(count, (unsigned long long)c);
}

// Single CTA, in place: w[b] holds the drawn leaf value and becomes (min_b' w[b'] / w[b])^beta = (N P_b)^-beta
// normalised by its batch maximum.  The min is order-independent, so the weights do not depend on the thread
// schedule and the smallest leaf of the batch gets exactly 1.  Every index is read and written by the same thread.
// A leaf of 0 (only an all-zero tree can hand one out) gets weight 1 and takes no part in the min.
constexpr int IS_WEIGHT_THREADS = 256;
__global__ void __launch_bounds__(IS_WEIGHT_THREADS) is_weight_kernel(float* __restrict__ w, int batch, float beta) {
  __shared__ float s_min[IS_WEIGHT_THREADS / 32];
  float m = INFINITY;
  for (int b = threadIdx.x; b < batch; b += blockDim.x)
    if (w[b] > 0.f) m = fminf(m, w[b]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fminf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) s_min[threadIdx.x >> 5] = m;
  __syncthreads();
  m = s_min[0];
#pragma unroll
  for (int k = 1; k < IS_WEIGHT_THREADS / 32; ++k) m = fminf(m, s_min[k]);
  for (int b = threadIdx.x; b < batch; b += blockDim.x) {
    const float leaf = w[b];
    w[b] = (beta == 0.f || !(leaf > 0.f)) ? 1.0f : powf(__fdiv_rn(m, leaf), beta);
  }
}

__device__ __forceinline__ float node_sum(const float* __restrict__ children) {
  const float4* ch4 = reinterpret_cast<const float4*>(children);
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < TREE_K / 4; ++k) {
    const float4 v = ch4[k];
    s = __fadd_rn(s, v.x); s = __fadd_rn(s, v.y); s = __fadd_rn(s, v.z); s = __fadd_rn(s, v.w);
  }
  return s;
}

// single CTA: write the batch's leaves (highest batch index wins on duplicates, learner.py:136-139
// executes the writes in batch order), then refresh every ancestor level by level.  The leaf indices sit in shared
// memory: the last-writer test is a broadcast scan of the later entries (B^2 / 2 shared reads instead of global ones).
// kExponent: the shard stores p^alpha (r2d2_replay_set_priority_exponent); without it the leaf is prio[i] as given.
// kShardFilter (global sampling): the batch is the W*B records of all ranks in global-index order, published into
// this rank's exchange block; the kernel first waits for every rank's "records published" flag (`flags` + world words,
// `epoch`, expiry -> *status), then applies only the records whose shard is `owner` (the others take part as -1).
template <bool kExponent, bool kShardFilter = false>
__global__ void __launch_bounds__(1024) tree_update_kernel(TreeView tv, const long long* __restrict__ leaf,
                                                           const float* __restrict__ prio, int batch, float alpha,
                                                           const int* __restrict__ shard = nullptr, int owner = 0,
                                                           const unsigned* flags = nullptr, int world = 0,
                                                           unsigned epoch = 0, unsigned* status = nullptr) {
  extern __shared__ long long s_leaf[];
  if (kShardFilter) {
    if ((int)threadIdx.x < world) spin_until(flags + threadIdx.x, epoch, status);
    __syncthreads();
  }
  for (int i = threadIdx.x; i < batch; i += blockDim.x) {
    if (kShardFilter) s_leaf[i] = *reinterpret_cast<const volatile int*>(shard + i) == owner
                                      ? *reinterpret_cast<const volatile long long*>(leaf + i) : -1;
    else s_leaf[i] = leaf[i];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < batch; i += blockDim.x) {
    const long long li = s_leaf[i];
    if (kShardFilter && li < 0) continue;
    bool winner = true;
    for (int j = i + 1; j < batch; ++j)
      if (s_leaf[j] == li) { winner = false; break; }
    if (winner) {
      const float p = kShardFilter ? *reinterpret_cast<const volatile float*>(prio + i) : prio[i];
      if (kExponent) tv.lvl[0][li] = raise_priority(p, alpha);
      else tv.lvl[0][li] = p;
    }
  }
  __syncthreads();
  long long div = TREE_K;
  for (int l = 1; l < tv.levels; ++l) {
    for (int i = threadIdx.x; i < batch; i += blockDim.x) {
      if (kShardFilter && s_leaf[i] < 0) continue;
      const long long node = s_leaf[i] / div;
      tv.lvl[l][node] = node_sum(tv.lvl[l - 1] + node * TREE_K);
    }
    __syncthreads();
    div *= TREE_K;
  }
}

__global__ void __launch_bounds__(256) tree_recompute_range_kernel(TreeView tv, int level, long long first,
                                                                   long long count) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= count) return;
  const long long node = first + i;
  tv.lvl[level][node] = node_sum(tv.lvl[level - 1] + node * TREE_K);
}

// One launch gathers the whole time-major batch (replay_memory.py:116-133: slice, transpose, stack, H2D in the
// reference).  A warp owns one (t, b) pair: source row leaf[b] + t; it copies the obs row and the act row with
// lane-contiguous accesses (16-byte vectors when the row width is a multiple of 4 floats: a row start is then 16-byte
// aligned in both the shard and the batch), lane 0 moves the reward / terminal scalars.  Tasks >= T*B move the stored
// recurrent states: task T*B + nh*B + b copies state_rows[leaf[b]][nh][:] to out[nh][b][:].  No division per element.
// kPerDraw (global sampling): B counts the W*Bc global draws; draw b goes to rank b / Bc's slot (dst_base[b / Bc] plus
// the slot offsets), column b % Bc, and draws with leaf[b] < 0 belong to another shard and are skipped.
struct GatherParams {
  const float *obs_rows, *act_rows, *rew_rows, *term_rows;
  const void* state_rows;   // float, or __half under kHalfStates
  const long long* leaf;
  float *obs, *act, *rew, *term, *states;
  int T, B, O, A, H;
  int Bc;
  size_t off_obs, off_act, off_rew, off_term, off_states;
  GlobalPeers dst;
  const float *norm_mean, *norm_inv_std;   // kNormObs: the shard's observation normaliser (r2d2_replay_set_obs_normalizer)
  float norm_clip;
};

__device__ __forceinline__ void warp_copy_row(const float* __restrict__ src, float* __restrict__ dst, int n, int lane) {
  if ((n & 3) == 0) {
    const float4* s4 = reinterpret_cast<const float4*>(src);
    float4* d4 = reinterpret_cast<float4*>(dst);
    for (int k = lane; k < (n >> 2); k += 32) d4[k] = __ldg(s4 + k);
  } else {
    for (int k = lane; k < n; k += 32) dst[k] = __ldg(src + k);
  }
}

// warp_copy_row with the observation transform applied to every element (obs_norm_apply); feature k of the row reads
// mean[k] and inv_std[k], vectorised as the copy is.
__device__ __forceinline__ void warp_norm_row(const float* __restrict__ src, float* __restrict__ dst, int n, int lane,
                                              const float* __restrict__ mean, const float* __restrict__ inv_std,
                                              float clip) {
  if ((n & 3) == 0) {
    const float4* s4 = reinterpret_cast<const float4*>(src);
    const float4* m4 = reinterpret_cast<const float4*>(mean);
    const float4* i4 = reinterpret_cast<const float4*>(inv_std);
    float4* d4 = reinterpret_cast<float4*>(dst);
    for (int k = lane; k < (n >> 2); k += 32) {
      const float4 x = __ldg(s4 + k), m = __ldg(m4 + k), s = __ldg(i4 + k);
      d4[k] = make_float4(obs_norm_apply(x.x, m.x, s.x, clip), obs_norm_apply(x.y, m.y, s.y, clip),
                          obs_norm_apply(x.z, m.z, s.z, clip), obs_norm_apply(x.w, m.w, s.w, clip));
    }
  } else {
    for (int k = lane; k < n; k += 32) dst[k] = obs_norm_apply(__ldg(src + k), __ldg(mean + k), __ldg(inv_std + k), clip);
  }
}

// A stored fp16 state row widened into the fp32 batch (exact).  The sub-row starts at byte 2 H (8 leaf + nh) of the
// ring and at float H (nh ld + col) of the batch, so H % 8 == 0 makes 16-byte loads (8 halves -> two float4 stores)
// aligned at both ends, H % 4 == 0 8-byte loads (4 halves -> one float4 store); other widths go scalar.
__device__ __forceinline__ void warp_widen_row(const __half* __restrict__ src, float* __restrict__ dst, int n, int lane) {
  if ((n & 7) == 0) {
    const uint4* s8 = reinterpret_cast<const uint4*>(src);
    float4* d4 = reinterpret_cast<float4*>(dst);
    for (int k = lane; k < (n >> 3); k += 32) {
      const Float8 f = widen8(__ldg(s8 + k));
      d4[2 * k] = f.lo;
      d4[2 * k + 1] = f.hi;
    }
  } else if ((n & 3) == 0) {
    const uint2* s4 = reinterpret_cast<const uint2*>(src);
    float4* d4 = reinterpret_cast<float4*>(dst);
    for (int k = lane; k < (n >> 2); k += 32) d4[k] = widen4(__ldg(s4 + k));
  } else {
    for (int k = lane; k < n; k += 32) dst[k] = __half2float(src[k]);
  }
}

// Host-tier state rows (R2D2_STATE_MEMORY_HOST): the same sub-row copies, but every lane issues all its loads of a
// chunk before its first store, so a warp's whole request (2 KB of fp32 or 1 KB of fp16 states at H = 512: four or two
// 16-byte loads per lane) is in flight over the host link at once.  Plain loads: the rows are mapped host memory.
constexpr int kHostLoads = 4;   // loads in flight per lane

template <typename V>
__device__ __forceinline__ void load_chunk(const V* __restrict__ src, V (&v)[kHostLoads], int k0, int n, int lane) {
#pragma unroll
  for (int j = 0; j < kHostLoads; ++j) {
    const int k = k0 + j * 32 + lane;
    if (k < n) v[j] = src[k];
  }
}

__device__ __forceinline__ void host_copy_row(const float* __restrict__ src, float* __restrict__ dst, int n, int lane) {
  if ((n & 3) == 0) {
    const float4* s4 = reinterpret_cast<const float4*>(src);
    float4* d4 = reinterpret_cast<float4*>(dst);
    for (int k0 = 0; k0 < (n >> 2); k0 += 32 * kHostLoads) {
      float4 v[kHostLoads];
      load_chunk(s4, v, k0, n >> 2, lane);
#pragma unroll
      for (int j = 0; j < kHostLoads; ++j)
        if (k0 + j * 32 + lane < (n >> 2)) d4[k0 + j * 32 + lane] = v[j];
    }
  } else {
    for (int k0 = 0; k0 < n; k0 += 32 * kHostLoads) {
      float v[kHostLoads];
      load_chunk(src, v, k0, n, lane);
#pragma unroll
      for (int j = 0; j < kHostLoads; ++j)
        if (k0 + j * 32 + lane < n) dst[k0 + j * 32 + lane] = v[j];
    }
  }
}

// warp_widen_row's three routes (16-byte, 8-byte, scalar by H % 8 and H % 4) with the loads of a chunk first
__device__ __forceinline__ void host_widen_row(const __half* __restrict__ src, float* __restrict__ dst, int n, int lane) {
  if ((n & 7) == 0) {
    const uint4* s8 = reinterpret_cast<const uint4*>(src);
    float4* d4 = reinterpret_cast<float4*>(dst);
    for (int k0 = 0; k0 < (n >> 3); k0 += 32 * kHostLoads) {
      uint4 v[kHostLoads];
      load_chunk(s8, v, k0, n >> 3, lane);
#pragma unroll
      for (int j = 0; j < kHostLoads; ++j) {
        const int k = k0 + j * 32 + lane;
        if (k < (n >> 3)) {
          const Float8 f = widen8(v[j]);
          d4[2 * k] = f.lo;
          d4[2 * k + 1] = f.hi;
        }
      }
    }
  } else if ((n & 3) == 0) {
    const uint2* s4 = reinterpret_cast<const uint2*>(src);
    float4* d4 = reinterpret_cast<float4*>(dst);
    for (int k0 = 0; k0 < (n >> 2); k0 += 32 * kHostLoads) {
      uint2 v[kHostLoads];
      load_chunk(s4, v, k0, n >> 2, lane);
#pragma unroll
      for (int j = 0; j < kHostLoads; ++j)
        if (k0 + j * 32 + lane < (n >> 2)) d4[k0 + j * 32 + lane] = widen4(v[j]);
    }
  } else {
    for (int k0 = 0; k0 < n; k0 += 32 * kHostLoads) {
      __half v[kHostLoads];
      load_chunk(src, v, k0, n, lane);
#pragma unroll
      for (int j = 0; j < kHostLoads; ++j)
        if (k0 + j * 32 + lane < n) dst[k0 + j * 32 + lane] = __half2float(v[j]);
    }
  }
}

// kHalfStates: state_rows holds __half (r2d2_replay_options.state_storage = R2D2_STATE_F16); the batch stays fp32.
// kHostStates (R2D2_STATE_MEMORY_HOST): state_rows is mapped host memory.  The 8 B state tasks then come FIRST (task
// nh * B + b; row task t * B + b follows at 8 B + t * B + b), so that every host read is in flight from the start of the
// launch and overlaps the HBM row copies instead of adding a host round trip after them; the row tasks are unchanged.
// The two tiers are separate kernels (gather_batch_kernel and gather_host_states_kernel) over this one body.
// kNormObs: the obs rows go through the shard's observation normaliser (the *_norm_kernel instantiations).
template <bool kPerDraw, bool kHalfStates, bool kHostStates, bool kNormObs>
__device__ __forceinline__ void gather_batch(GatherParams g) {
  const int lane = threadIdx.x & 31;
  const long long warp0 = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  const long long row_tasks = (long long)g.T * g.B;
  const long long total = row_tasks + (g.states ? (long long)8 * g.B : 0);
  const int lead = kHostStates && g.states ? 8 : 0;                       // state "rows" before the row tasks
  int t = (int)(warp0 / g.B), b = (int)(warp0 % g.B);                    // one division per warp, then carried
  const int dt = (int)(n_warps / g.B), db = (int)(n_warps % g.B);
  for (long long task = warp0; task < total; task += n_warps) {
    // destination of draw b: the batch's own buffers, column b of B; per draw, rank b / Bc's slot, column b % Bc
    const long long leaf = g.leaf[b];
    float *obs = g.obs, *act = g.act, *rew = g.rew, *term = g.term, *states = g.states;
    int col = b, ld = g.B;
    if (kPerDraw) {
      char* d = g.dst.base[b / g.Bc];
      obs = reinterpret_cast<float*>(d + g.off_obs); act = reinterpret_cast<float*>(d + g.off_act);
      rew = reinterpret_cast<float*>(d + g.off_rew); term = reinterpret_cast<float*>(d + g.off_term);
      states = reinterpret_cast<float*>(d + g.off_states);
      col = b % g.Bc; ld = g.Bc;
    }
    if (kPerDraw && leaf < 0) {
      // another shard's draw
    } else if (kHostStates ? t >= lead : task < row_tasks) {
      const long long r = leaf + (t - lead);
      const long long o = (long long)(t - lead) * ld + col;
      if (obs) {
        if (kNormObs) warp_norm_row(g.obs_rows + r * g.O, obs + o * g.O, g.O, lane, g.norm_mean, g.norm_inv_std, g.norm_clip);
        else warp_copy_row(g.obs_rows + r * g.O, obs + o * g.O, g.O, lane);
      }
      if (act) warp_copy_row(g.act_rows + r * g.A, act + o * g.A, g.A, lane);
      if (lane == 0) {
        if (rew) rew[o] = __ldg(g.rew_rows + r);
        if (term) term[o] = __ldg(g.term_rows + r);
      }
    } else if (kHostStates) {
      if (kHalfStates)
        host_widen_row(static_cast<const __half*>(g.state_rows) + (leaf * 8 + t) * g.H,
                       states + ((long long)t * ld + col) * g.H, g.H, lane);
      else
        host_copy_row(static_cast<const float*>(g.state_rows) + (leaf * 8 + t) * g.H,
                      states + ((long long)t * ld + col) * g.H, g.H, lane);
    } else if (kHalfStates) {
      warp_widen_row(static_cast<const __half*>(g.state_rows) + (leaf * 8 + (t - g.T)) * g.H,
                     states + ((long long)(t - g.T) * ld + col) * g.H, g.H, lane);
    } else {
      warp_copy_row(static_cast<const float*>(g.state_rows) + (leaf * 8 + (t - g.T)) * g.H,
                    states + ((long long)(t - g.T) * ld + col) * g.H, g.H, lane);
    }
    t += dt; b += db;
    if (b >= g.B) { b -= g.B; ++t; }
  }
}

template <bool kPerDraw = false, bool kHalfStates = false>
__global__ void __launch_bounds__(256) gather_batch_kernel(GatherParams g) {
  gather_batch<kPerDraw, kHalfStates, false, false>(g);
}

template <bool kPerDraw = false, bool kHalfStates = false>
__global__ void __launch_bounds__(256) gather_host_states_kernel(GatherParams g) {
  gather_batch<kPerDraw, kHalfStates, true, false>(g);
}

template <bool kPerDraw = false, bool kHalfStates = false>
__global__ void __launch_bounds__(256) gather_batch_norm_kernel(GatherParams g) {
  gather_batch<kPerDraw, kHalfStates, false, true>(g);
}

template <bool kPerDraw = false, bool kHalfStates = false>
__global__ void __launch_bounds__(256) gather_host_states_norm_kernel(GatherParams g) {
  gather_batch<kPerDraw, kHalfStates, true, true>(g);
}

// ---- observation moments at ingest (r2d2_replay_add_episodes_ex) ----
// Per ring run, right after its copy: a row counts when it is no pad row and all its O values are finite; then two
// passes over a fixed partition of the run's rows into chunks of kMomChunk - the sums (mean), then the squared
// deviations from that mean (M2) - with one double partial per (chunk, feature), added in chunk order by one CTA.  No
// floating-point atomics: the bits do not depend on the schedule.
constexpr int kMomChunk = 128;

// valid[i] = keep[i] && every obs value of row i is finite, one warp per row, grid-stride over the rows (the grid is
// capped: a run may have any number of rows); kept rows that are not finite are counted (integer atomics, one per row).
__global__ void __launch_bounds__(256) obs_row_valid_kernel(const float* __restrict__ obs, const unsigned char* __restrict__ keep,
                                                            long long n, int O, unsigned char* __restrict__ valid,
                                                            unsigned long long* __restrict__ n_bad) {
  const int lane = threadIdx.x & 31;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long row = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5; row < n; row += n_warps) {   // warp-uniform
    bool fin = true;
    for (int k = lane; k < O; k += 32) fin = fin && isfinite(obs[row * O + k]);
    fin = __all_sync(0xffffffffu, fin);
    if (lane == 0) {
      const bool kept = keep[row] != 0;
      valid[row] = kept && fin;
      if (kept && !fin) atomicAdd(n_bad, 1ull);
    }
  }
}

// grid (chunks, ceil(O / 32)), block (32, 8): thread (x, y) sums feature 32 by + x over rows y, y + 8, .. of chunk bx,
// then the 8 row groups are added in order.  The chunk index is the x dimension, so a run of up to 2^31 - 1 chunks fits
// one launch.  kSquares: (x - mean)^2 instead of x.  Pass 1 also counts the chunk's rows.
template <bool kSquares>
__global__ void __launch_bounds__(256) obs_moment_partial_kernel(const float* __restrict__ obs,
                                                                 const unsigned char* __restrict__ valid, long long n,
                                                                 int O, const double* __restrict__ mean,
                                                                 double* __restrict__ part, int* __restrict__ count) {
  __shared__ double s[8][33];
  const int o = blockIdx.y * 32 + threadIdx.x;
  const long long r0 = (long long)blockIdx.x * kMomChunk, r1 = min(n, r0 + kMomChunk);
  double acc = 0.0;
  if (o < O) {
    const double m = kSquares ? mean[o] : 0.0;
    for (long long r = r0 + threadIdx.y; r < r1; r += 8) {
      if (!valid[r]) continue;
      const double x = (double)obs[r * O + o];
      if (kSquares) {
        const double d = __dsub_rn(x, m);
        acc = __dadd_rn(acc, __dmul_rn(d, d));
      } else {
        acc = __dadd_rn(acc, x);
      }
    }
  }
  s[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0 && o < O) {
    double t = s[0][threadIdx.x];
#pragma unroll
    for (int k = 1; k < 8; ++k) t = __dadd_rn(t, s[k][threadIdx.x]);
    part[blockIdx.x * (long long)O + o] = t;
  }
  if (!kSquares && blockIdx.y == 0 && threadIdx.x == 0 && threadIdx.y == 0) {
    int c = 0;
    for (long long r = r0; r < r1; ++r) c += valid[r];
    count[blockIdx.x] = c;
  }
}

// One CTA.  Pass 1: the run's count and mean into run[0], run[1 .. O].  Pass 2: the run's M2, and the run merged into
// the call's block `acc` (Chan, chan_merge).
template <bool kSquares>
__global__ void __launch_bounds__(256) obs_moment_finish_kernel(const double* __restrict__ part,
                                                                const int* __restrict__ count, int chunks, int O,
                                                                double* __restrict__ run, double* __restrict__ acc) {
  long long c = 0;
  for (int k = 0; k < chunks; ++k) c += count[k];
  const double nb = (double)c, na = kSquares ? acc[0] : 0.0;
  for (int o = threadIdx.x; o < O; o += blockDim.x) {
    double t = 0.0;
    for (int k = 0; k < chunks; ++k) t = __dadd_rn(t, part[(long long)k * O + o]);
    if (!kSquares) {
      run[1 + o] = c ? __ddiv_rn(t, nb) : 0.0;
    } else {
      double m = acc[1 + o], m2 = acc[1 + O + o];
      chan_merge(na, m, m2, nb, run[1 + o], t);
      acc[1 + o] = m;
      acc[1 + O + o] = m2;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    if (kSquares) acc[0] = __dadd_rn(na, nb);
    else run[0] = nb;
  }
}

int grid_for(long long total) {
  long long blocks = (total + 255) / 256;
  if (blocks > num_sms() * 16) blocks = num_sms() * 16;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

}  // namespace

struct Episode {
  long long row_start;
  int n_rows;
  int n_starts;
  long long serial;
};

struct Replay {
  r2d2_replay_config cfg;
  int rows_per_window;
  float *obs_rows = nullptr, *act_rows = nullptr, *rew_rows = nullptr, *term_rows = nullptr;
  // The recurrent states [cap,4,2,H]: fp32, or __half under R2D2_STATE_F16 (half_states).  In HBM, or under
  // R2D2_STATE_MEMORY_HOST (host_states) in mapped, page-locked host memory (host_alloc, freed with cudaFreeHost) that
  // state_rows addresses through its device pointer.  Rows: state_row_bytes / state_row.
  char* state_rows = nullptr;
  bool half_states = false;
  bool host_states = false;
  void* host_alloc = nullptr;
  size_t host_bytes = 0;
  // grow-only device staging block (stage_states): [count (16 B) | the packed states of the largest call so far]
  char* stage = nullptr;
  size_t stage_bytes = 0;
  // grow-only device scratch of the ingest moments: [n_bad (16 B) | run block 1 + O | partials | counts | keep | valid]
  char* mom = nullptr;
  size_t mom_bytes = 0;
  size_t device_bytes = 0;   // every device allocation of the shard (rows, tree, staging, moment scratch)
  // observation normaliser of every gather (r2d2_replay_set_obs_normalizer): DEVICE [O] each, NULL = raw obs
  const float* norm_mean = nullptr;
  const float* norm_inv_std = nullptr;
  float norm_clip = 0.f;
  std::vector<float*> level_alloc;
  TreeView tv;
  std::deque<Episode> episodes;
  std::map<long long, long long> by_row;  // row_start -> serial
  long long next_serial = 0;
  long long head = 0;
  long long sequence_counter = 0;
  long long rows_used = 0;
  long long evicted_total = 0;
  float alpha = 1.0f;   // priority exponent: leaves hold p^alpha (1 = the raw priority, no pow on any path)
  struct Group {        // global sampling (r2d2_replay_attach_group)
    int rank = 0, world = 1, batch = 0;
    GlobalPeers peers{};
    GlobalLayout lay;
    unsigned wb_epoch = 0, draw_epoch = 0;
    int wb_stage = 0, draw_stage = 0;   // next stage of the write-back / draw that is in progress
    bool drawn_since_wb = true;         // a write-back needs a draw since the last one (the record block is reused)
  };
  Group* group = nullptr;
  struct Import {       // a snapshot restore between r2d2_replay_import_begin and _end
    struct Run { long long src, dst, n; };   // packed snapshot rows [src, src + n) -> ring rows [dst, dst + n)
    std::vector<Run> runs;
    std::vector<Episode> kept;               // at their ring rows, FIFO order
    std::vector<long long> kept_src;         // packed snapshot row of each kept episode
    long long packed_rows = 0, received = 0;
    int storage = R2D2_STATE_F32;            // the snapshot's state storage
    long long head = 0, sequence_counter = 0, next_serial = 0, evicted_total = 0, rows_used = 0;
  };
  Import* import = nullptr;
};

// bytes of one [4,2,H] state row stored as fp16 (half) or fp32, or in the shard's type; the address of ring row i
static size_t state_row_bytes(const Replay* r, bool half) {
  return (half ? sizeof(__half) : sizeof(float)) * 8 * (size_t)r->cfg.hidden;
}
static size_t state_row_bytes(const Replay* r) { return state_row_bytes(r, r->half_states); }
static char* state_row(const Replay* r, long long i) { return r->state_rows + i * state_row_bytes(r); }

static int recompute_ancestors(Replay* r, long long first_leaf, long long n_leaves, cudaStream_t stream) {
  long long lo = first_leaf, hi = first_leaf + n_leaves - 1;
  for (int l = 1; l < r->tv.levels; ++l) {
    lo /= TREE_K;
    hi /= TREE_K;
    const long long count = hi - lo + 1;
    tree_recompute_range_kernel<<<(int)((count + 255) / 256), 256, 0, stream>>>(r->tv, l, lo, count);
    count_launch();
  }
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

int replay_create(Replay** out, const r2d2_replay_config* cfg, const r2d2_replay_options* options) {
  R2D2_REQUIRE(out && cfg, "null");
  R2D2_REQUIRE(cfg->obs_size > 0 && cfg->n_actions > 0 && cfg->hidden > 0, "sizes");
  R2D2_REQUIRE(cfg->capacity_rows > 0, "capacity_rows");
  const r2d2_replay_options opt = options ? *options : r2d2_replay_options{};   // zeroed = fp32 states in HBM
  R2D2_REQUIRE(opt.state_storage == R2D2_STATE_F32 || opt.state_storage == R2D2_STATE_F16,
               "state_storage is R2D2_STATE_F32 or R2D2_STATE_F16");
  R2D2_REQUIRE(opt.state_memory == R2D2_STATE_MEMORY_DEVICE || opt.state_memory == R2D2_STATE_MEMORY_HOST,
               "state_memory is R2D2_STATE_MEMORY_DEVICE or R2D2_STATE_MEMORY_HOST");
  Replay* r = new Replay();
  r->cfg = *cfg;
  r->rows_per_window = cfg->burn_in + cfg->learning + cfg->n_step;
  r->half_states = opt.state_storage == R2D2_STATE_F16;
  r->host_states = opt.state_memory == R2D2_STATE_MEMORY_HOST;
  const long long cap = cfg->capacity_rows;
  const size_t state_bytes = (size_t)cap * state_row_bytes(r);
  if (r->host_states) {   // first, so that a refusal leaves nothing allocated
    void* dev = nullptr;
    cudaError_t e = cudaHostAlloc(&r->host_alloc, state_bytes, cudaHostAllocMapped | cudaHostAllocPortable);
    if (e == cudaSuccess) e = cudaHostGetDevicePointer(&dev, r->host_alloc, 0);
    if (e != cudaSuccess) {
      cudaGetLastError();
      if (r->host_alloc) cudaFreeHost(r->host_alloc);
      delete r;
      set_last_error("replay shard: " + std::to_string(state_bytes) + " bytes of mapped pinned host memory for the "
                     "recurrent states could not be allocated (" + cudaGetErrorString(e) + ")");
      return R2D2_ERR_CUDA;
    }
    memset(r->host_alloc, 0, state_bytes);   // nothing can be in flight on a buffer that was just allocated
    r->host_bytes = state_bytes;
    r->state_rows = static_cast<char*>(dev);
  }
  auto dmalloc_bytes = [&](void** p, size_t bytes) -> int {
    R2D2_CUDA_TRY(cudaMalloc(p, bytes));
    R2D2_CUDA_TRY(cudaMemset(*p, 0, bytes));
    r->device_bytes += bytes;
    return R2D2_OK;
  };
  auto dmalloc = [&](float** p, long long n) -> int {
    return dmalloc_bytes(reinterpret_cast<void**>(p), sizeof(float) * (size_t)n);
  };
  int rc = R2D2_OK;
  if ((rc = dmalloc(&r->obs_rows, cap * cfg->obs_size)) || (rc = dmalloc(&r->act_rows, cap * cfg->n_actions)) ||
      (rc = dmalloc(&r->rew_rows, cap)) || (rc = dmalloc(&r->term_rows, cap)) ||
      (!r->host_states && (rc = dmalloc_bytes(reinterpret_cast<void**>(&r->state_rows), state_bytes)))) {
    replay_destroy(r);
    return rc;
  }
  // levels: n[0] = leaves, n[l+1] = ceil(n[l]/32), last level has one node (the total)
  long long n = (cap + TREE_K - 1) / TREE_K * TREE_K;
  int levels = 0;
  while (true) {
    R2D2_REQUIRE(levels < TREE_MAX_LEVELS, "tree too deep");
    const long long parents = (n + TREE_K - 1) / TREE_K;
    const long long alloc = (n > 1) ? parents * TREE_K : TREE_K;
    float* p = nullptr;
    if ((rc = dmalloc(&p, alloc))) { replay_destroy(r); return rc; }
    r->level_alloc.push_back(p);
    r->tv.lvl[levels] = p;
    r->tv.n[levels] = n;
    ++levels;
    if (n == 1) break;
    n = parents;
  }
  r->tv.levels = levels;
  *out = r;
  return R2D2_OK;
}

int replay_set_priority_exponent(Replay* r, float alpha) {
  R2D2_REQUIRE(r, "null");
  R2D2_REQUIRE(alpha >= 0.f && alpha <= 1.f, "priority exponent must lie in [0, 1]");
  if (!r->episodes.empty()) {   // raw and exponentiated leaves in one tree would silently skew the draw
    set_last_error("the priority exponent can only be set while the replay shard holds no episode");
    return R2D2_ERR_STATE;
  }
  r->alpha = alpha;
  return R2D2_OK;
}

// leaves [first, first + n) were just copied from the host as raw priorities: store p^alpha instead
static int raise_fresh_leaves(Replay* r, long long first, long long n, cudaStream_t stream) {
  if (r->alpha == 1.0f || n <= 0) return R2D2_OK;
  raise_leaves_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(r->tv.lvl[0] + first, n, r->alpha);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

// The staging block starts with a count (fp16 overflow at ingest, bad leaves at restore); the packed states follow 16
// bytes in, so every packed row of 8 H values starts 16-byte aligned, as the conversion kernels need.
constexpr size_t kStageHead = 16;

static int ensure_stage(Replay* r, size_t need) {
  if (need > r->stage_bytes) {
    R2D2_CUDA_TRY(cudaFree(r->stage));   // synchronises: no conversion of an earlier call still reads the old block
    r->stage = nullptr;
    r->device_bytes -= r->stage_bytes;
    r->stage_bytes = 0;
    R2D2_CUDA_TRY(cudaMalloc(&r->stage, need));
    r->stage_bytes = need;
    r->device_bytes += need;
  }
  return R2D2_OK;
}

// The packed state rows of an ingest or restore call, as store_states reads them: the caller's host buffer, or the
// staging block (which holds zeros past the caller's rows).
struct StateSource {
  const char* base;   // packed row 0
  bool half;          // fp16 rows, else fp32
  bool staged;
};

// The call's n_src packed state rows (fp16 or fp32, host memory) go through the staging block if and only if the shard
// keeps its states in host memory - every write to the mapped rows is then stream-ordered device work - or in the other
// type, whose conversion kernel reads device memory.  Staged, they are zero-padded to n_rows rows, and fp32 states
// bound for fp16 rows are range-checked: a finite value that fp16 would round to +-inf refuses the whole call with
// R2D2_ERR_ARG before anything is placed, evicted or committed (one stream synchronisation: the count is read on the
// host).  Unstaged, the source is the caller's buffer.
static int stage_states(Replay* r, const void* states, bool half, long long n_src, long long n_rows, cudaStream_t stream,
                        StateSource* out) {
  *out = {static_cast<const char*>(states), half, false};
  if (!r->host_states && half == r->half_states) return R2D2_OK;
  const size_t row = state_row_bytes(r, half);
  R2D2_TRY(ensure_stage(r, kStageHead + row * (size_t)n_rows));
  char* staged = r->stage + kStageHead;
  *out = {staged, half, true};
  if (n_src > 0) R2D2_CUDA_TRY(cudaMemcpyAsync(staged, states, row * (size_t)n_src, cudaMemcpyHostToDevice, stream));
  if (n_rows > n_src) R2D2_CUDA_TRY(cudaMemsetAsync(staged + row * n_src, 0, row * (size_t)(n_rows - n_src), stream));
  if (half || !r->half_states) return R2D2_OK;
  const long long n = n_src * 8LL * r->cfg.hidden;
  unsigned long long* d_count = reinterpret_cast<unsigned long long*>(r->stage);
  R2D2_CUDA_TRY(cudaMemsetAsync(d_count, 0, sizeof(*d_count), stream));
  if (n > 0) {
    count_f16_overflow_kernel<<<grid_for(n), 256, 0, stream>>>(reinterpret_cast<const float*>(staged), n, d_count);
    count_launch();
    R2D2_CUDA_TRY(cudaGetLastError());
  }
  unsigned long long count = 0;
  R2D2_CUDA_TRY(cudaMemcpyAsync(&count, d_count, sizeof(count), cudaMemcpyDeviceToHost, stream));
  R2D2_CUDA_TRY(cudaStreamSynchronize(stream));
  if (count) {
    set_last_error(std::to_string(count) + " finite recurrent-state value(s) of magnitude >= 65520 would round to "
                   "+-inf in fp16 state storage: nothing of this call was stored");
    return R2D2_ERR_ARG;
  }
  return R2D2_OK;
}

// Packed rows [src_row, src_row + n_rows) of `src` into ring rows [ring_row, ring_row + n_rows): one copy when the types
// match (cudaMemcpyDefault: either end may be host memory), else one rounding or widening kernel, which also stores
// straight into mapped host rows.
static int store_states(Replay* r, long long ring_row, const StateSource& src, long long src_row, long long n_rows,
                        cudaStream_t stream) {
  if (n_rows <= 0) return R2D2_OK;
  const char* from = src.base + src_row * state_row_bytes(r, src.half);
  char* to = state_row(r, ring_row);
  if (src.half == r->half_states) {
    R2D2_CUDA_TRY(cudaMemcpyAsync(to, from, state_row_bytes(r, src.half) * (size_t)n_rows, cudaMemcpyDefault, stream));
    return R2D2_OK;
  }
  const long long n = n_rows * 8LL * r->cfg.hidden;
  if (r->half_states)
    states_to_f16_kernel<<<grid_for(n / 8), 256, 0, stream>>>(reinterpret_cast<const float*>(from),
                                                              reinterpret_cast<__half*>(to), n);
  else
    states_from_f16_kernel<<<grid_for(n / 8), 256, 0, stream>>>(reinterpret_cast<const __half*>(from),
                                                                reinterpret_cast<float*>(to), n);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

// Packed host rows [src_row, src_row + n_rows) of obs / act / rew / term into ring rows [ring_row, ring_row + n_rows),
// and the first n_state_rows of them from the states of `src`.  The leaves stay with the callers.
static int write_rows(Replay* r, long long ring_row, long long src_row, long long n_rows, const float* obs,
                      const float* act, const float* rew, const float* term, const StateSource& src,
                      long long n_state_rows, cudaStream_t stream) {
  const size_t O = r->cfg.obs_size, A = r->cfg.n_actions, n = (size_t)n_rows;
  R2D2_CUDA_TRY(cudaMemcpyAsync(r->obs_rows + ring_row * O, obs + src_row * O, sizeof(float) * n * O,
                                cudaMemcpyHostToDevice, stream));
  R2D2_CUDA_TRY(cudaMemcpyAsync(r->act_rows + ring_row * A, act + src_row * A, sizeof(float) * n * A,
                                cudaMemcpyHostToDevice, stream));
  R2D2_CUDA_TRY(cudaMemcpyAsync(r->rew_rows + ring_row, rew + src_row, sizeof(float) * n, cudaMemcpyHostToDevice, stream));
  R2D2_CUDA_TRY(cudaMemcpyAsync(r->term_rows + ring_row, term + src_row, sizeof(float) * n, cudaMemcpyHostToDevice,
                                stream));
  return store_states(r, ring_row, src, src_row, n_state_rows, stream);
}

int replay_destroy(Replay* r) {
  if (!r) return R2D2_OK;
  cudaFree(r->obs_rows); cudaFree(r->act_rows); cudaFree(r->rew_rows); cudaFree(r->term_rows);
  if (r->host_states) cudaFreeHost(r->host_alloc);
  else cudaFree(r->state_rows);
  cudaFree(r->stage);
  cudaFree(r->mom);
  for (float* p : r->level_alloc) cudaFree(p);
  delete r->group;
  delete r->import;
  delete r;
  return R2D2_OK;
}

// Ranges of leaves whose ancestors must be refreshed; merged and recomputed once per ingest call.
typedef std::vector<std::pair<long long, long long>> RangeList;   // (first leaf, count)

static int refresh_ranges(Replay* r, RangeList& ranges, cudaStream_t stream) {
  if (ranges.empty()) return R2D2_OK;
  std::sort(ranges.begin(), ranges.end());
  long long lo = ranges[0].first, hi = ranges[0].first + ranges[0].second;
  for (size_t i = 1; i <= ranges.size(); ++i) {
    // merge ranges that share a parent node (distance < fan-out): one launch chain instead of two
    if (i < ranges.size() && ranges[i].first <= hi + TREE_K) {
      hi = std::max(hi, ranges[i].first + ranges[i].second);
      continue;
    }
    R2D2_TRY(recompute_ancestors(r, lo, hi - lo, stream));
    if (i < ranges.size()) { lo = ranges[i].first; hi = ranges[i].first + ranges[i].second; }
  }
  ranges.clear();
  return R2D2_OK;
}

static int evict_front(Replay* r, cudaStream_t stream, RangeList* deferred) {
  const Episode e = r->episodes.front();
  r->episodes.pop_front();
  r->by_row.erase(e.row_start);
  // replay_memory.py:149: the counter drops by len(episode) - sequence_length (sic: not the amount added at :147)
  r->sequence_counter -= e.n_rows - (r->cfg.burn_in + r->cfg.learning);
  r->rows_used -= e.n_rows;
  ++r->evicted_total;
  if (e.n_starts > 0) {
    R2D2_CUDA_TRY(cudaMemsetAsync(r->tv.lvl[0] + e.row_start, 0, sizeof(float) * e.n_starts, stream));
    if (deferred) deferred->push_back({e.row_start, (long long)e.n_starts});
    else R2D2_TRY(recompute_ancestors(r, e.row_start, e.n_starts, stream));
  }
  return R2D2_OK;
}

// Ring placement of an episode of n_rows rows: wrap when the tail gap is too small, then evict - oldest first, the
// reference's FIFO order (replay_memory.py:148-152) - until no live episode overlaps [start, start + n_rows).  After a
// wrap the oldest episode may sit at the TAIL of the ring while a younger one occupies the head that is about to be
// overwritten: evicting from the front until the overlap is gone removes both (ADVICE r1: the earlier loop stopped at
// the first non-overlapping front episode and then failed the overlap check).
static int place_episode(Replay* r, int n_rows, cudaStream_t stream, RangeList* deferred, long long* start_out) {
  R2D2_REQUIRE(n_rows <= r->cfg.capacity_rows, "episode larger than the ring");
  if (r->head + n_rows > r->cfg.capacity_rows) r->head = 0;  // wrap: the tail gap stays unused
  const long long start = r->head, end = start + n_rows;
  auto overlaps = [&]() {
    for (const Episode& e : r->episodes)
      if (e.row_start < end && start < e.row_start + e.n_rows) return true;
    return false;
  };
  while (!r->episodes.empty() && overlaps()) R2D2_TRY(evict_front(r, stream, deferred));
  *start_out = start;
  return R2D2_OK;
}

static void commit_episode(Replay* r, long long start, int n_rows, int n_starts) {
  Episode e{start, n_rows, n_starts, r->next_serial++};
  r->episodes.push_back(e);
  r->by_row[start] = e.serial;
  r->head = start + n_rows;
  r->rows_used += n_rows;
  r->sequence_counter += n_rows - (r->rows_per_window - 1);  // replay_memory.py:147
}

// The end of an ingest call: the cap's evictions (replay_memory.py:148-152), one refresh of every touched leaf range,
// and the synchronisation after which the caller may release its host buffers.
static int finish_ingest(Replay* r, RangeList& ranges, cudaStream_t stream) {
  while (r->cfg.max_sequences > 0 && r->sequence_counter > r->cfg.max_sequences && !r->episodes.empty())
    R2D2_TRY(evict_front(r, stream, &ranges));
  R2D2_TRY(refresh_ranges(r, ranges, stream));
  R2D2_CUDA_TRY(cudaStreamSynchronize(stream));
  return R2D2_OK;
}

int replay_add_episode(Replay* r, const float* obs, const float* act, const float* rew, const float* term,
                       const float* states, int n_rows, int n_state_rows, const float* priority, int n_starts,
                       cudaStream_t stream) {
  R2D2_REQUIRE(r && obs && act && rew && term && states, "null");
  R2D2_REQUIRE(n_rows >= r->rows_per_window, "episode shorter than one window");
  R2D2_REQUIRE(n_starts >= 0 && n_starts <= n_rows - r->rows_per_window + 1, "n_starts exceeds valid window starts");
  R2D2_REQUIRE(n_state_rows >= n_starts && n_state_rows <= n_rows, "state rows");
  R2D2_REQUIRE(n_starts == 0 || priority, "priority");
  StateSource src;
  R2D2_TRY(stage_states(r, states, false, n_state_rows, n_rows, stream, &src));
  RangeList ranges;
  long long start = 0;
  R2D2_TRY(place_episode(r, n_rows, stream, &ranges, &start));
  // rows past n_state_rows get zero states: staged, the block holds them; from the caller's buffer, a memset
  const long long n_stored = src.staged ? n_rows : n_state_rows;
  R2D2_TRY(write_rows(r, start, 0, n_rows, obs, act, rew, term, src, n_stored, stream));
  if (n_stored < n_rows)
    R2D2_CUDA_TRY(cudaMemsetAsync(state_row(r, start + n_stored), 0, state_row_bytes(r) * (size_t)(n_rows - n_stored), stream));
  if (n_starts > 0) {
    R2D2_CUDA_TRY(cudaMemcpyAsync(r->tv.lvl[0] + start, priority, sizeof(float) * (size_t)n_starts,
                                  cudaMemcpyHostToDevice, stream));
    R2D2_TRY(raise_fresh_leaves(r, start, n_starts, stream));
  }
  if (n_rows > n_starts)
    R2D2_CUDA_TRY(cudaMemsetAsync(r->tv.lvl[0] + start + n_starts, 0, sizeof(float) * (size_t)(n_rows - n_starts), stream));
  ranges.push_back({start, (long long)n_rows});
  commit_episode(r, start, n_rows, n_starts);
  return finish_ingest(r, ranges, stream);
}

// One actor file at a time (LearnerReplayMemory.load, replay_memory.py:138-157): every episode of the file is appended,
// THEN the oldest episodes are dropped while the sequence counter exceeds the cap - the reference's order.  The rows
// of all episodes arrive packed ([R, *] with R = sum of n_rows; recurrent states zero-padded to R rows, leaf
// priorities already expanded to one value per row): contiguous runs in the ring are one copy per tensor, the sum tree
// is refreshed once over the merged touched ranges, and there is one stream synchronisation per file.
// The moments of ring rows [ring_row, ring_row + n) - packed rows [first, first + n) of the call - merged into the
// call's block: kernels of the ingest moments above, reading the keep flags the caller staged in the scratch.
struct MomentScratch {
  unsigned long long* n_bad;
  double *run, *part;
  int* count;
  unsigned char *keep, *valid;
};

static int run_moments(Replay* r, const MomentScratch& m, long long ring_row, long long first, long long n,
                       double* acc, cudaStream_t stream) {
  if (n <= 0) return R2D2_OK;
  const int O = r->cfg.obs_size;
  const float* obs = r->obs_rows + ring_row * O;
  const int chunks = (int)((n + kMomChunk - 1) / kMomChunk);
  obs_row_valid_kernel<<<grid_for(n * 32), 256, 0, stream>>>(obs, m.keep + first, n, O, m.valid, m.n_bad);
  const dim3 grid((unsigned)chunks, (unsigned)ceil_div(O, 32)), block(32, 8);
  obs_moment_partial_kernel<false><<<grid, block, 0, stream>>>(obs, m.valid, n, O, nullptr, m.part, m.count);
  obs_moment_finish_kernel<false><<<1, 256, 0, stream>>>(m.part, m.count, chunks, O, m.run, acc);
  obs_moment_partial_kernel<true><<<grid, block, 0, stream>>>(obs, m.valid, n, O, m.run + 1, m.part, m.count);
  obs_moment_finish_kernel<true><<<1, 256, 0, stream>>>(m.part, m.count, chunks, O, m.run, acc);
  count_launch(5);
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

int replay_add_episodes(Replay* r, int n_episodes, const int* n_rows, const int* n_starts, const float* obs,
                        const float* act, const float* rew, const float* term, const float* states,
                        const float* leaf_prio, long long* row_start_out, long long* n_evicted_out,
                        long long* sequence_counter_out, cudaStream_t stream, double* obs_moments,
                        long long* n_nonfinite_out) {
  R2D2_REQUIRE(r && n_episodes >= 0 && (n_episodes == 0 || (n_rows && n_starts && obs && act && rew && term && states && leaf_prio)),
               "null");
  long long R = 0;
  for (int e = 0; e < n_episodes; ++e) {
    R2D2_REQUIRE(n_rows[e] >= r->rows_per_window, "episode shorter than one window");
    R2D2_REQUIRE(n_starts[e] >= 0 && n_starts[e] <= n_rows[e] - r->rows_per_window + 1, "n_starts exceeds valid window starts");
    R2D2_REQUIRE(n_rows[e] <= r->cfg.capacity_rows, "episode larger than the ring");
    R += n_rows[e];
  }
  StateSource src{};
  if (n_episodes > 0) R2D2_TRY(stage_states(r, states, false, R, R, stream, &src));
  // obs_moments: the keep flags of the call's rows (0 on each episode's last n_step rows, the actors' pad rows) are
  // staged next to the moment scratch; the block starts empty and every ring run is merged into it after its copy
  MomentScratch ms{};
  std::vector<unsigned char> keep;
  if (obs_moments) {
    const int O = r->cfg.obs_size;
    const long long chunks = (R + kMomChunk - 1) / kMomChunk;
    auto up = [](size_t x) { return (x + 255) / 256 * 256; };
    const size_t o_run = 256, o_part = up(o_run + sizeof(double) * (1 + (size_t)O)),
                 o_count = up(o_part + sizeof(double) * (size_t)chunks * O), o_keep = up(o_count + sizeof(int) * chunks),
                 o_valid = up(o_keep + (size_t)R), need = up(o_valid + (size_t)R);
    if (need > r->mom_bytes) {
      R2D2_CUDA_TRY(cudaFree(r->mom));   // synchronises: no earlier call's moments still read the old block
      r->mom = nullptr;
      r->device_bytes -= r->mom_bytes;
      r->mom_bytes = 0;
      R2D2_CUDA_TRY(cudaMalloc(&r->mom, need));
      r->mom_bytes = need;
      r->device_bytes += need;
    }
    ms = {reinterpret_cast<unsigned long long*>(r->mom), reinterpret_cast<double*>(r->mom + o_run),
          reinterpret_cast<double*>(r->mom + o_part), reinterpret_cast<int*>(r->mom + o_count),
          reinterpret_cast<unsigned char*>(r->mom + o_keep), reinterpret_cast<unsigned char*>(r->mom + o_valid)};
    keep.assign((size_t)R, 1);
    long long off = 0;
    for (int e = 0; e < n_episodes; ++e) {
      for (int k = n_rows[e] - r->cfg.n_step; k < n_rows[e]; ++k) keep[(size_t)(off + k)] = 0;
      off += n_rows[e];
    }
    R2D2_CUDA_TRY(cudaMemsetAsync(r->mom, 0, sizeof(unsigned long long), stream));
    R2D2_CUDA_TRY(cudaMemsetAsync(obs_moments, 0, sizeof(double) * (1 + 2 * (size_t)O), stream));
    if (R > 0) R2D2_CUDA_TRY(cudaMemcpyAsync(ms.keep, keep.data(), (size_t)R, cudaMemcpyHostToDevice, stream));
  }
  const long long evicted0 = r->evicted_total;
  RangeList ranges;
  long long first = 0;                  // first packed row of the current run
  long long run_start = -1, run_rows = 0;
  auto flush = [&]() -> int {
    if (run_rows == 0) return R2D2_OK;
    R2D2_TRY(write_rows(r, run_start, first, run_rows, obs, act, rew, term, src, run_rows, stream));
    // a later run of the same call may overwrite these rows (a call wider than the ring): the moments are taken now
    if (obs_moments) R2D2_TRY(run_moments(r, ms, run_start, first, run_rows, obs_moments, stream));
    R2D2_CUDA_TRY(cudaMemcpyAsync(r->tv.lvl[0] + run_start, leaf_prio + first, sizeof(float) * (size_t)run_rows,
                                  cudaMemcpyHostToDevice, stream));
    R2D2_TRY(raise_fresh_leaves(r, run_start, run_rows, stream));
    ranges.push_back({run_start, run_rows});
    first += run_rows;
    run_rows = 0;
    return R2D2_OK;
  };
  for (int e = 0; e < n_episodes; ++e) {
    // A placement that wraps starts a new run, and its evictions may hit episodes of the pending run: their leaves are
    // zeroed by a memset that has to follow the run's copy, so the run is flushed before the placement.  Without a wrap
    // the episode lands right after the run and overlaps none of it.
    if (r->head + n_rows[e] > r->cfg.capacity_rows) R2D2_TRY(flush());
    long long start = 0;
    R2D2_TRY(place_episode(r, n_rows[e], stream, &ranges, &start));
    if (run_rows == 0) run_start = start;
    run_rows += n_rows[e];
    commit_episode(r, start, n_rows[e], n_starts[e]);
    if (row_start_out) row_start_out[e] = start;
  }
  R2D2_TRY(flush());
  unsigned long long n_bad = 0;
  if (obs_moments) R2D2_CUDA_TRY(cudaMemcpyAsync(&n_bad, ms.n_bad, sizeof(n_bad), cudaMemcpyDeviceToHost, stream));
  R2D2_TRY(finish_ingest(r, ranges, stream));
  if (n_nonfinite_out) *n_nonfinite_out = (long long)n_bad;
  if (n_evicted_out) *n_evicted_out = r->evicted_total - evicted0;
  if (sequence_counter_out) *sequence_counter_out = r->sequence_counter;
  return R2D2_OK;
}

// The ring side of a gather: the shard's rows and sizes.  The caller fills in the leaves and the destination.
static GatherParams ring_gather_params(const Replay* r) {
  GatherParams g{};
  g.obs_rows = r->obs_rows; g.act_rows = r->act_rows; g.rew_rows = r->rew_rows; g.term_rows = r->term_rows;
  g.state_rows = r->state_rows;
  g.T = r->rows_per_window; g.O = r->cfg.obs_size; g.A = r->cfg.n_actions; g.H = r->cfg.hidden;
  g.norm_mean = r->norm_mean; g.norm_inv_std = r->norm_inv_std; g.norm_clip = r->norm_clip;
  return g;
}

// The gather instantiation for the shard's state type and tier, one warp per task
template <bool kPerDraw>
static int launch_gather(const Replay* r, const GatherParams& g, long long tasks, cudaStream_t stream) {
  const int grid = grid_for(tasks * 32);
  if (r->norm_mean) {
    if (r->host_states && r->half_states) gather_host_states_norm_kernel<kPerDraw, true><<<grid, 256, 0, stream>>>(g);
    else if (r->host_states) gather_host_states_norm_kernel<kPerDraw, false><<<grid, 256, 0, stream>>>(g);
    else if (r->half_states) gather_batch_norm_kernel<kPerDraw, true><<<grid, 256, 0, stream>>>(g);
    else gather_batch_norm_kernel<kPerDraw, false><<<grid, 256, 0, stream>>>(g);
  } else if (r->host_states && r->half_states) gather_host_states_kernel<kPerDraw, true><<<grid, 256, 0, stream>>>(g);
  else if (r->host_states) gather_host_states_kernel<kPerDraw, false><<<grid, 256, 0, stream>>>(g);
  else if (r->half_states) gather_batch_kernel<kPerDraw, true><<<grid, 256, 0, stream>>>(g);
  else gather_batch_kernel<kPerDraw, false><<<grid, 256, 0, stream>>>(g);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

int replay_set_obs_normalizer(Replay* r, const float* mean_f, const float* inv_std_f, float clip) {
  R2D2_REQUIRE(r, "null");
  R2D2_REQUIRE((mean_f == nullptr) == (inv_std_f == nullptr), "mean_f and inv_std_f are both given or both NULL");
  R2D2_REQUIRE(!mean_f || (clip > 0.f && clip <= FLT_MAX), "clip must be finite and > 0");
  R2D2_REQUIRE(!mean_f || (r->cfg.obs_size % 4 != 0 ||
                           ((reinterpret_cast<uintptr_t>(mean_f) | reinterpret_cast<uintptr_t>(inv_std_f)) & 15) == 0),
               "mean_f and inv_std_f must be 16-byte aligned when obs_size is a multiple of 4");
  r->norm_mean = mean_f;
  r->norm_inv_std = inv_std_f;
  r->norm_clip = mean_f ? clip : 0.f;
  return R2D2_OK;
}

int replay_device_bytes(Replay* r, size_t* out) {
  R2D2_REQUIRE(r && out, "null");
  *out = r->device_bytes;
  return R2D2_OK;
}

int replay_host_bytes(Replay* r, size_t* out) {
  R2D2_REQUIRE(r && out, "null");
  *out = r->host_bytes;
  return R2D2_OK;
}

int replay_gather(Replay* r, const long long* leaf_idx, int batch, float* obs, float* act, float* rew, float* term,
                  float* states, cudaStream_t stream) {
  R2D2_REQUIRE(r && leaf_idx && batch > 0, "args");
  if (!(obs || act || rew || term || states)) {
    R2D2_CUDA_TRY(cudaGetLastError());
    return R2D2_OK;
  }
  GatherParams g = ring_gather_params(r);
  g.leaf = leaf_idx;
  g.obs = obs; g.act = act; g.rew = rew; g.term = term; g.states = states;
  g.B = batch;
  return launch_gather<false>(r, g, (long long)g.T * batch + (states ? (long long)8 * batch : 0), stream);
}

int replay_sample(Replay* r, const float* u, int batch, long long* leaf_idx, float* obs, float* act, float* rew,
                  float* term, float* states, cudaStream_t stream) {
  R2D2_REQUIRE(r && u && leaf_idx && batch > 0, "args");
  R2D2_REQUIRE(!r->episodes.empty(), "replay is empty");
  tree_sample_kernel<false><<<ceil_div(batch, 256), 256, 0, stream>>>(r->tv, u, batch, leaf_idx, nullptr);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return replay_gather(r, leaf_idx, batch, obs, act, rew, term, states, stream);
}

int replay_sample_weighted(Replay* r, const float* u, int batch, float beta, long long* leaf_idx, float* is_weight,
                           float* obs, float* act, float* rew, float* term, float* states, cudaStream_t stream) {
  R2D2_REQUIRE(r && u && leaf_idx && is_weight && batch > 0, "args");
  R2D2_REQUIRE(beta >= 0.f && beta <= 1.f, "importance-sampling exponent must lie in [0, 1]");
  R2D2_REQUIRE(!r->episodes.empty(), "replay is empty");
  tree_sample_kernel<true><<<ceil_div(batch, 256), 256, 0, stream>>>(r->tv, u, batch, leaf_idx, is_weight);
  count_launch();
  is_weight_kernel<<<1, IS_WEIGHT_THREADS, 0, stream>>>(is_weight, batch, beta);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return replay_gather(r, leaf_idx, batch, obs, act, rew, term, states, stream);
}

int replay_update_priorities(Replay* r, const long long* leaf_idx, const float* prio, int batch, cudaStream_t stream) {
  R2D2_REQUIRE(r && leaf_idx && prio && batch > 0, "args");
  R2D2_REQUIRE(batch <= 5120, "priority batch larger than the shared-memory index table (40 KB)");
  if (r->alpha == 1.0f)
    tree_update_kernel<false><<<1, 1024, sizeof(long long) * (size_t)batch, stream>>>(r->tv, leaf_idx, prio, batch, 1.0f);
  else
    tree_update_kernel<true><<<1, 1024, sizeof(long long) * (size_t)batch, stream>>>(r->tv, leaf_idx, prio, batch, r->alpha);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

int replay_stats(Replay* r, r2d2_replay_stats_t* out, cudaStream_t stream) {
  R2D2_REQUIRE(r && out, "args");
  float total = 0.f;
  R2D2_CUDA_TRY(cudaMemcpyAsync(&total, r->tv.lvl[r->tv.levels - 1], sizeof(float), cudaMemcpyDeviceToHost, stream));
  R2D2_CUDA_TRY(cudaStreamSynchronize(stream));
  out->n_episodes = (long long)r->episodes.size();
  out->n_rows_used = r->rows_used;
  out->sequence_counter = r->sequence_counter;
  out->capacity_rows = r->cfg.capacity_rows;
  out->tree_levels = r->tv.levels;
  long long nodes = 0;
  for (int l = 0; l < r->tv.levels; ++l) nodes += r->tv.n[l];
  out->tree_nodes = nodes;
  out->last_row_start = r->episodes.empty() ? -1 : r->episodes.back().row_start;
  out->total_priority = total;
  return R2D2_OK;
}

int replay_decode(Replay* r, const long long* leaf_host, int n, long long* episode_index, long long* sequence_index) {
  R2D2_REQUIRE(r && leaf_host && episode_index && sequence_index, "args");
  const long long front_serial = r->episodes.empty() ? 0 : r->episodes.front().serial;
  for (int i = 0; i < n; ++i) {
    episode_index[i] = sequence_index[i] = -1;
    auto it = r->by_row.upper_bound(leaf_host[i]);
    if (it == r->by_row.begin()) continue;
    --it;
    const Episode& e = r->episodes[(size_t)(it->second - front_serial)];
    if (leaf_host[i] < e.row_start + e.n_rows) {
      episode_index[i] = it->second - front_serial;
      sequence_index[i] = leaf_host[i] - e.row_start;
    }
  }
  return R2D2_OK;
}

int replay_tree_level(Replay* r, int level, const float** dev_ptr, long long* n) {
  R2D2_REQUIRE(r && level >= 0 && level < r->tv.levels, "level");
  *dev_ptr = r->tv.lvl[level];
  *n = r->tv.n[level];
  return R2D2_OK;
}

// ---- snapshots (r2d2_replay_export_* / r2d2_replay_import_*) ----------------------------------------------------------
// The live episodes' rows, their leaves and the host bookkeeping are the whole state of a shard: every other leaf is 0
// (ingest and evict_front zero them) and every tree node is the left-to-right sum of its children, so a full rebuild
// from the leaves gives every level back bit for bit.

int replay_export_info(Replay* r, r2d2_replay_snapshot_info* out) {
  R2D2_REQUIRE(r && out, "null");
  const r2d2_replay_config& c = r->cfg;
  out->obs_size = c.obs_size; out->n_actions = c.n_actions; out->hidden = c.hidden;
  out->burn_in = c.burn_in; out->learning = c.learning; out->n_step = c.n_step;
  out->state_storage = r->half_states ? R2D2_STATE_F16 : R2D2_STATE_F32;
  out->priority_exponent = r->alpha;
  out->capacity_rows = c.capacity_rows; out->max_sequences = c.max_sequences;
  out->n_episodes = (long long)r->episodes.size();
  out->head = r->head; out->sequence_counter = r->sequence_counter; out->next_serial = r->next_serial;
  out->evicted_total = r->evicted_total; out->rows_used = r->rows_used;
  return R2D2_OK;
}

int replay_export_episodes(Replay* r, long long* row_start, int* n_rows, int* n_starts, long long* serial) {
  R2D2_REQUIRE(r && (r->episodes.empty() || (row_start && n_rows && n_starts && serial)), "null");
  size_t i = 0;
  for (const Episode& e : r->episodes) {
    row_start[i] = e.row_start; n_rows[i] = e.n_rows; n_starts[i] = e.n_starts; serial[i] = e.serial;
    ++i;
  }
  return R2D2_OK;
}

int replay_export_rows(Replay* r, long long first, long long n, float* obs, float* act, float* rew, float* term,
                       void* states, float* leaves, cudaStream_t stream) {
  R2D2_REQUIRE(r && obs && act && rew && term && states && leaves, "null");
  R2D2_REQUIRE(first >= 0 && n >= 0 && first + n <= r->cfg.capacity_rows, "row range outside the ring");
  const size_t O = r->cfg.obs_size, A = r->cfg.n_actions, k = (size_t)n;
  R2D2_CUDA_TRY(cudaMemcpyAsync(obs, r->obs_rows + first * O, sizeof(float) * k * O, cudaMemcpyDeviceToHost, stream));
  R2D2_CUDA_TRY(cudaMemcpyAsync(act, r->act_rows + first * A, sizeof(float) * k * A, cudaMemcpyDeviceToHost, stream));
  R2D2_CUDA_TRY(cudaMemcpyAsync(rew, r->rew_rows + first, sizeof(float) * k, cudaMemcpyDeviceToHost, stream));
  R2D2_CUDA_TRY(cudaMemcpyAsync(term, r->term_rows + first, sizeof(float) * k, cudaMemcpyDeviceToHost, stream));
  // cudaMemcpyDefault: the host tier's rows are host memory.  Only ingest and restore write them, and both synchronise
  // the stream before they return, so no write to these rows is in flight here
  R2D2_CUDA_TRY(cudaMemcpyAsync(states, state_row(r, first), state_row_bytes(r) * k, cudaMemcpyDefault, stream));
  R2D2_CUDA_TRY(cudaMemcpyAsync(leaves, r->tv.lvl[0] + first, sizeof(float) * k, cudaMemcpyDeviceToHost, stream));
  R2D2_CUDA_TRY(cudaStreamSynchronize(stream));
  return R2D2_OK;
}

// A refused restore leaves the shard empty: no episode, zero counters, every tree node 0.
static void abandon_import(Replay* r, cudaStream_t stream) {
  delete r->import;
  r->import = nullptr;
  r->episodes.clear();
  r->by_row.clear();
  r->head = r->sequence_counter = r->next_serial = r->evicted_total = r->rows_used = 0;
  for (int l = 0; l < r->tv.levels; ++l) cudaMemsetAsync(r->tv.lvl[l], 0, sizeof(float) * (size_t)r->tv.n[l], stream);
  cudaStreamSynchronize(stream);
}

static int refuse_import(Replay* r, cudaStream_t stream, const std::string& why) {
  abandon_import(r, stream);
  set_last_error("replay snapshot refused, the shard is left empty: " + why);
  return R2D2_ERR_ARG;
}

int replay_import_begin(Replay* r, const r2d2_replay_snapshot_info* info, const long long* row_start,
                        const int* n_rows, const int* n_starts, const long long* serial, long long* n_dropped_out,
                        cudaStream_t stream) {
  R2D2_REQUIRE(r && info, "null");
  R2D2_REQUIRE(info->n_episodes == 0 || (row_start && n_rows && n_starts && serial), "null episode table");
  if (!r->episodes.empty() || r->import) {
    set_last_error("a replay snapshot can only be restored into an empty shard");
    return R2D2_ERR_STATE;
  }
  const r2d2_replay_config& c = r->cfg;
  auto refuse = [&](const std::string& why) { return refuse_import(r, stream, why); };
  if (info->obs_size != c.obs_size || info->n_actions != c.n_actions || info->hidden != c.hidden ||
      info->burn_in != c.burn_in || info->learning != c.learning || info->n_step != c.n_step)
    return refuse("the snapshot's obs / act / hidden / burn-in / learning / n-step (" + std::to_string(info->obs_size) +
                  " " + std::to_string(info->n_actions) + " " + std::to_string(info->hidden) + " " +
                  std::to_string(info->burn_in) + " " + std::to_string(info->learning) + " " +
                  std::to_string(info->n_step) + ") differ from the shard's (" + std::to_string(c.obs_size) + " " +
                  std::to_string(c.n_actions) + " " + std::to_string(c.hidden) + " " + std::to_string(c.burn_in) +
                  " " + std::to_string(c.learning) + " " + std::to_string(c.n_step) + ")");
  if (info->priority_exponent != r->alpha)
    return refuse("the snapshot's leaves hold p^" + std::to_string(info->priority_exponent) + ", the shard stores p^" +
                  std::to_string(r->alpha) + " (the raw priorities are not kept)");
  if (info->state_storage != R2D2_STATE_F32 && info->state_storage != R2D2_STATE_F16)
    return refuse("unknown state storage " + std::to_string(info->state_storage));
  if (info->n_episodes < 0 || info->capacity_rows <= 0 || info->head < 0 || info->head > info->capacity_rows)
    return refuse("bad counters");
  // the episode table: valid episodes, consecutive serials (decode indexes the FIFO by serial), disjoint ring ranges
  Replay::Import* im = new Replay::Import();
  r->import = im;
  std::vector<std::pair<long long, long long>> spans;
  long long total = 0;
  for (long long e = 0; e < info->n_episodes; ++e) {
    if (n_rows[e] < r->rows_per_window || n_starts[e] < 0 || n_starts[e] > n_rows[e] - r->rows_per_window + 1 ||
        row_start[e] < 0 || row_start[e] + n_rows[e] > info->capacity_rows || serial[e] != serial[0] + e)
      return refuse("episode " + std::to_string(e) + " of the table is malformed");
    spans.push_back({row_start[e], row_start[e] + n_rows[e]});
    total += n_rows[e];
  }
  std::sort(spans.begin(), spans.end());
  for (size_t i = 1; i < spans.size(); ++i)
    if (spans[i].first < spans[i - 1].second) return refuse("episodes of the table overlap in the ring");
  if (total != info->rows_used || (info->n_episodes > 0 && info->next_serial != serial[info->n_episodes - 1] + 1))
    return refuse("the episode table does not match the counters");
  im->packed_rows = total;
  im->sequence_counter = info->sequence_counter;
  im->next_serial = info->next_serial;
  im->evicted_total = info->evicted_total;
  im->rows_used = total;
  const bool same = info->capacity_rows == c.capacity_rows;
  long long first_kept = 0, dropped = 0;
  if (!same) {   // compacted from row 0 in FIFO order; the oldest go while the rest does not fit (evict_front's counts)
    while (first_kept < info->n_episodes && im->rows_used > c.capacity_rows) {
      im->sequence_counter -= n_rows[first_kept] - (c.burn_in + c.learning);
      im->rows_used -= n_rows[first_kept];
      ++im->evicted_total;
      ++first_kept;
      ++dropped;
    }
  }
  long long src = 0, dst = 0;
  for (long long e = 0; e < info->n_episodes; ++e) {
    if (e >= first_kept) {
      const long long at = same ? row_start[e] : dst;
      im->kept.push_back(Episode{at, n_rows[e], n_starts[e], serial[e]});
      im->kept_src.push_back(src);
      if (!im->runs.empty() && im->runs.back().src + im->runs.back().n == src && im->runs.back().dst + im->runs.back().n == at)
        im->runs.back().n += n_rows[e];
      else
        im->runs.push_back({src, at, (long long)n_rows[e]});
      dst = at + n_rows[e];
    }
    src += n_rows[e];
  }
  im->head = same ? info->head : dst;
  im->storage = info->state_storage;
  // leaves outside the restored episodes must be 0 for the rebuild; a fresh shard already has them so
  R2D2_CUDA_TRY(cudaMemsetAsync(r->tv.lvl[0], 0, sizeof(float) * (size_t)r->tv.n[0], stream));
  if (n_dropped_out) *n_dropped_out = dropped;
  return R2D2_OK;
}

int replay_import_rows(Replay* r, long long first, long long n, const float* obs, const float* act, const float* rew,
                       const float* term, const void* states, const float* leaves, cudaStream_t stream) {
  R2D2_REQUIRE(r && obs && act && rew && term && states && leaves, "null");
  if (!r->import) { set_last_error("r2d2_replay_import_rows without r2d2_replay_import_begin"); return R2D2_ERR_STATE; }
  Replay::Import& im = *r->import;
  if (first != im.received || n <= 0 || first + n > im.packed_rows)
    return refuse_import(r, stream, "rows [" + std::to_string(first) + ", " + std::to_string(first + n) +
                                        ") do not continue the " + std::to_string(im.received) + " of " +
                                        std::to_string(im.packed_rows) + " rows received so far");
  StateSource src;   // the file's states (in its type), staged as ingest stages them
  const int rc = stage_states(r, states, im.storage == R2D2_STATE_F16, n, n, stream, &src);
  if (rc == R2D2_ERR_ARG) return refuse_import(r, stream, std::string(last_error()));
  R2D2_TRY(rc);
  R2D2_TRY(ensure_stage(r, kStageHead));   // the bad-leaf count
  unsigned long long* d_count = reinterpret_cast<unsigned long long*>(r->stage);
  R2D2_CUDA_TRY(cudaMemsetAsync(d_count, 0, sizeof(*d_count), stream));
  for (const Replay::Import::Run& run : im.runs) {
    const long long lo = std::max(run.src, first), hi = std::min(run.src + run.n, first + n);
    if (lo >= hi) continue;
    const long long s = lo - first, d = run.dst + (lo - run.src), k = hi - lo;
    R2D2_TRY(write_rows(r, d, s, k, obs, act, rew, term, src, k, stream));
    R2D2_CUDA_TRY(cudaMemcpyAsync(r->tv.lvl[0] + d, leaves + s, sizeof(float) * (size_t)k, cudaMemcpyHostToDevice, stream));
  }
  for (size_t e = 0; e < im.kept.size(); ++e) {   // every kept episode's piece of this chunk: its leaves checked
    const Episode& ep = im.kept[e];
    const long long lo = std::max(im.kept_src[e], first), hi = std::min(im.kept_src[e] + ep.n_rows, first + n);
    if (lo >= hi) continue;
    const long long valid = std::max(0LL, std::min(hi, im.kept_src[e] + ep.n_starts) - lo);
    count_bad_leaves_kernel<<<grid_for(hi - lo), 256, 0, stream>>>(r->tv.lvl[0] + ep.row_start + (lo - im.kept_src[e]),
                                                                   hi - lo, valid, d_count);
    count_launch();
    R2D2_CUDA_TRY(cudaGetLastError());
  }
  unsigned long long bad = 0;
  R2D2_CUDA_TRY(cudaMemcpyAsync(&bad, d_count, sizeof(bad), cudaMemcpyDeviceToHost, stream));
  R2D2_CUDA_TRY(cudaStreamSynchronize(stream));   // the caller may refill its host buffers
  if (bad)
    return refuse_import(r, stream, std::to_string(bad) + " leaf value(s) are negative, NaN or infinite, or nonzero on a "
                                    "row that starts no sequence");
  im.received += n;
  return R2D2_OK;
}

int replay_import_end(Replay* r, cudaStream_t stream) {
  R2D2_REQUIRE(r, "null");
  if (!r->import) { set_last_error("r2d2_replay_import_end without r2d2_replay_import_begin"); return R2D2_ERR_STATE; }
  Replay::Import& im = *r->import;
  if (im.received != im.packed_rows)
    return refuse_import(r, stream, "only " + std::to_string(im.received) + " of " + std::to_string(im.packed_rows) +
                                        " rows arrived");
  R2D2_TRY(recompute_ancestors(r, 0, r->cfg.capacity_rows, stream));
  for (const Episode& e : im.kept) {
    r->episodes.push_back(e);
    r->by_row[e.row_start] = e.serial;
  }
  r->head = im.head;
  r->sequence_counter = im.sequence_counter;
  r->next_serial = im.next_serial;
  r->evicted_total = im.evicted_total;
  r->rows_used = im.rows_used;
  delete r->import;
  r->import = nullptr;
  R2D2_CUDA_TRY(cudaStreamSynchronize(stream));
  return R2D2_OK;
}

GlobalLayout global_layout(int T, int B, int O, int A, int H, int world) {
  GlobalLayout l;
  const size_t n = (size_t)world * B;
  auto up = [](size_t x) { return (x + 255) / 256 * 256; };
  size_t off = 512;
  l.off_uniforms = off; off = up(off + sizeof(float) * n);
  l.off_rec_leaf = off; off = up(off + sizeof(long long) * n);
  l.off_rec_shard = off; off = up(off + sizeof(int) * n);
  l.off_rec_prio = off; off = up(off + sizeof(float) * n);
  l.off_draw_leaf = off; off = up(off + sizeof(long long) * n);
  l.exchange_bytes = off;
  off = 0;
  l.off_obs = off; off = up(off + sizeof(float) * (size_t)T * B * O);
  l.off_act = off; off = up(off + sizeof(float) * (size_t)T * B * A);
  l.off_rew = off; off = up(off + sizeof(float) * (size_t)T * B);
  l.off_term = off; off = up(off + sizeof(float) * (size_t)T * B);
  l.off_states = off; off = up(off + sizeof(float) * (size_t)8 * B * H);
  l.off_leaf = off; off = up(off + sizeof(long long) * B);
  l.off_shard = off; off = up(off + sizeof(int) * B);
  l.off_weight = off; off = up(off + sizeof(float) * B);
  l.off_slot_uniforms = off; off = up(off + sizeof(float) * B);
  l.slot_bytes = off;
  l.bytes = l.exchange_bytes + 2 * l.slot_bytes;
  return l;
}

int replay_attach_group(Replay* r, int rank, int world, int batch, void* const* peer_bases, size_t buffer_bytes) {
  R2D2_REQUIRE(r && peer_bases, "null argument");
  R2D2_REQUIRE(world >= 1 && world <= kGlobalMaxWorld && rank >= 0 && rank < world, "global sampling rank / world");
  R2D2_REQUIRE(batch > 0 && (long long)world * batch <= 5120,
               "global batch W * B must lie in [1, 5120] (the write-back's shared-memory index table)");
  R2D2_REQUIRE(!r->group, "replay shard already attached to a group");
  Replay::Group* g = new Replay::Group();
  g->rank = rank; g->world = world; g->batch = batch;
  g->lay = global_layout(r->rows_per_window, batch, r->cfg.obs_size, r->cfg.n_actions, r->cfg.hidden, world);
  if (buffer_bytes != g->lay.bytes) {   // the buffers were laid out for another shape: peer stores would miss
    delete g;
    set_last_error("global sampling buffer size does not match this shard's layout (rows, obs, act, hidden, batch, "
                   "world): the engine and the replay shard disagree");
    return R2D2_ERR_ARG;
  }
  for (int k = 0; k < world; ++k) {
    if (!peer_bases[k]) { delete g; R2D2_REQUIRE(false, "null peer buffer"); }
    g->peers.base[k] = static_cast<char*>(peer_bases[k]);
  }
  r->group = g;
  return R2D2_OK;
}

// stage 0: publish this rank's B records into every rank's exchange block; stage 1: wait for every rank's records and
// apply those that land in this shard (highest global index wins); -1: both.
int replay_global_write_back(Replay* r, int stage, const long long* leaf, const int* shard, const float* prio,
                             cudaStream_t stream) {
  R2D2_REQUIRE(r && r->group, "replay shard is not attached to a group");
  R2D2_REQUIRE(stage >= -1 && stage <= 1, "write-back stage is 0, 1 or -1 (both)");
  Replay::Group& g = *r->group;
  if (stage <= 0) {
    R2D2_REQUIRE(leaf && shard && prio, "null record");
    if (g.wb_stage != 0 || !g.drawn_since_wb) {
      set_last_error("a global write-back needs a global draw since the previous one, and its stages in order");
      return R2D2_ERR_STATE;
    }
    g.wb_epoch += 1;
    R2D2_TRY(global_publish_records(g.peers, g.lay, g.world, g.rank, g.batch, leaf, shard, prio, g.wb_epoch, stream));
    g.wb_stage = 1;
    g.drawn_since_wb = false;
  }
  if (stage == 1 || stage == -1) {
    if (g.wb_stage != 1) { set_last_error("write-back stage 1 before stage 0"); return R2D2_ERR_STATE; }
    char* own = g.peers.base[g.rank];
    const int n = g.world * g.batch;
    const long long* rl = reinterpret_cast<const long long*>(own + g.lay.off_rec_leaf);
    const int* rs = reinterpret_cast<const int*>(own + g.lay.off_rec_shard);
    const float* rp = reinterpret_cast<const float*>(own + g.lay.off_rec_prio);
    unsigned* flags = reinterpret_cast<unsigned*>(own);
    const size_t smem = sizeof(long long) * (size_t)n;
    if (r->alpha == 1.0f)
      tree_update_kernel<false, true><<<1, 1024, smem, stream>>>(r->tv, rl, rp, n, 1.0f, rs, g.rank, flags + kGlobalFlagPub,
                                                                 g.world, g.wb_epoch, flags + kGlobalStatus);
    else
      tree_update_kernel<true, true><<<1, 1024, smem, stream>>>(r->tv, rl, rp, n, r->alpha, rs, g.rank, flags + kGlobalFlagPub,
                                                                g.world, g.wb_epoch, flags + kGlobalStatus);
    count_launch();
    R2D2_CUDA_TRY(cudaGetLastError());
    g.wb_stage = 0;
  }
  return R2D2_OK;
}

// stage 0: publish this shard's root and this rank's B uniforms (fill slot `slot`) to every rank; stage 1: wait for
// every rank's root, draw all W*B, gather this shard's draws into the consumers' slots and signal delivery; stage 2:
// wait for every owner's delivery and form the importance weights; -1: all three.
int replay_global_draw(Replay* r, int stage, int slot, int weighted, float beta, cudaStream_t stream) {
  R2D2_REQUIRE(r && r->group, "replay shard is not attached to a group");
  R2D2_REQUIRE(stage >= -1 && stage <= 2, "draw stage is 0, 1, 2 or -1 (all)");
  R2D2_REQUIRE(slot == 0 || slot == 1, "batch slot");
  R2D2_REQUIRE(weighted == 0 || weighted == 1, "weighted is 0 or 1");
  R2D2_REQUIRE(beta >= 0.f && beta <= 1.f, "importance-sampling exponent must lie in [0, 1]");
  Replay::Group& g = *r->group;
  const bool all = stage == -1;
  if (all || stage == 0) {
    if (g.draw_stage != 0 || g.wb_stage != 0) {
      set_last_error("a global draw needs the previous draw and write-back complete, and its stages in order");
      return R2D2_ERR_STATE;
    }
    g.draw_epoch += 1;
    R2D2_TRY(global_publish_root(g.peers, g.lay, g.world, g.rank, g.batch, slot, r->tv.lvl[r->tv.levels - 1],
                                 g.draw_epoch, stream));
    g.draw_stage = 1;
  }
  if (all || stage == 1) {
    if (g.draw_stage != 1) { set_last_error("draw stage 1 out of order"); return R2D2_ERR_STATE; }
    if (weighted)
      global_draw_kernel<true><<<1, 1024, 0, stream>>>(r->tv, g.peers, g.lay, g.world, g.rank, g.batch, slot, g.draw_epoch);
    else
      global_draw_kernel<false><<<1, 1024, 0, stream>>>(r->tv, g.peers, g.lay, g.world, g.rank, g.batch, slot, g.draw_epoch);
    count_launch();
    R2D2_CUDA_TRY(cudaGetLastError());
    GatherParams gp = ring_gather_params(r);
    char* own = g.peers.base[g.rank];
    gp.leaf = reinterpret_cast<const long long*>(own + g.lay.off_draw_leaf);
    gp.states = reinterpret_cast<float*>(own + g.lay.slot(slot) + g.lay.off_states);   // non-null: state tasks run
    gp.B = g.world * g.batch; gp.Bc = g.batch;
    const size_t so = g.lay.slot(slot);
    gp.off_obs = so + g.lay.off_obs; gp.off_act = so + g.lay.off_act; gp.off_rew = so + g.lay.off_rew;
    gp.off_term = so + g.lay.off_term; gp.off_states = so + g.lay.off_states;
    gp.dst = g.peers;
    R2D2_TRY(launch_gather<true>(r, gp, (long long)(gp.T + 8) * gp.B, stream));
    R2D2_TRY(global_deliver(g.peers, g.world, g.rank, g.draw_epoch, stream));
    g.draw_stage = 2;
  }
  if (all || stage == 2) {
    if (g.draw_stage != 2) { set_last_error("draw stage 2 out of order"); return R2D2_ERR_STATE; }
    R2D2_TRY(global_receive(g.peers, g.lay, g.world, g.rank, g.batch, slot, weighted != 0, beta, g.draw_epoch, stream));
    g.draw_stage = 0;
    g.drawn_since_wb = true;
  }
  return R2D2_OK;
}

int replay_global_status(Replay* r, int* out, cudaStream_t stream) {
  R2D2_REQUIRE(r && r->group && out, "replay shard is not attached to a group");
  unsigned v = 0;
  R2D2_CUDA_TRY(cudaMemcpyAsync(&v, r->group->peers.base[r->group->rank] + sizeof(unsigned) * kGlobalStatus,
                                sizeof(unsigned), cudaMemcpyDeviceToHost, stream));
  R2D2_CUDA_TRY(cudaStreamSynchronize(stream));
  *out = (int)v;
  return R2D2_OK;
}

}  // namespace r2d2

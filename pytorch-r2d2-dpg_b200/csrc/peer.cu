// Gradient exchange over NVLink peer memory - see peer.cuh.
#include "peer.cuh"
#include "peer_sync.cuh"

namespace r2d2 {

namespace {

// flag words (uint32) inside the 4 KB flag area
constexpr int kFlagIn = 0;        // [2][16]  written by peer k at [block][k]: "gradients of iteration e complete"
constexpr int kFlagOut = 32;      // [2][16]  written by peer k at [block][k]: "my slice of iteration e is in your sums"
constexpr int kFlagCounter = 64;  // [2]      CTAs of the local reduce kernel that finished
constexpr int kFlagStatus = 66;   // [1]      1 = a bounded wait expired
// diagnostics (u64, byte offset 512): [0..1] ns the slice-sum kernel of block b waited for the peers' "gradients
// complete", [2..3] ns it ran in total, [4..5] ns the wait kernel of block b waited for "slice delivered", [6] start stamp
constexpr size_t kCounterBytes = 512;

__device__ __forceinline__ float4 ld_peer(const float4* p) {
  float4 v;
  asm volatile("ld.volatile.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
}

__global__ void peer_signal_kernel(PeerPtrs p, int world, int rank, size_t off_word, unsigned value) {
  const int k = threadIdx.x;
  if (k < world) {
    __threadfence_system();   // the gradient kernels ahead of this one in the stream happen-before the flag
    st_release_sys(reinterpret_cast<unsigned*>(p.base[k] + off_word) + rank, value);
  }
}

__global__ void peer_wait_kernel(const unsigned* flags, int world, unsigned value, unsigned* status,
                                 unsigned long long* waited_ns) {
  const unsigned long long t0 = global_ns();
  if ((int)threadIdx.x < world) spin_until(flags + threadIdx.x, value, status);
  __syncthreads();
  if (threadIdx.x == 0) *waited_ns += global_ns() - t0;
}

__global__ void __launch_bounds__(512)
peer_reduce_kernel(PeerPtrs p, int world, int rank, size_t off_flags, int block, size_t off_grads, size_t off_sums,
                   long long slice_vec, unsigned value) {
  unsigned* flags = reinterpret_cast<unsigned*>(p.base[rank] + off_flags);
  unsigned long long* counters = reinterpret_cast<unsigned long long*>(p.base[rank] + off_flags + kCounterBytes);
  const unsigned long long t0 = global_ns();
  if ((int)threadIdx.x < world) spin_until(flags + kFlagIn + block * kPeerMaxWorld + threadIdx.x, value, flags + kFlagStatus);
  __syncthreads();
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    counters[block] += global_ns() - t0;
    counters[6] = t0;
  }
  const long long first = (long long)rank * slice_vec;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < slice_vec; i += (long long)gridDim.x * blockDim.x) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int k0 = 0; k0 < world; k0 += 8) {   // rank order 0..world-1; 8 peer loads in flight per thread
      float4 v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (k0 + j < world) v[j] = ld_peer(reinterpret_cast<const float4*>(p.base[k0 + j] + off_grads) + first + i);
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (k0 + j < world) { acc.x += v[j].x; acc.y += v[j].y; acc.z += v[j].z; acc.w += v[j].w; }
    }
    for (int k = 0; k < world; ++k) reinterpret_cast<float4*>(p.base[k] + off_sums)[first + i] = acc;
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned* counter = flags + kFlagCounter + block;
    const unsigned done = atomicAdd(counter, 1u) + 1u;
    if (done == gridDim.x) {   // last CTA: every slice store of this rank is ordered before the flags
      *counter = 0u;
      counters[2 + block] += global_ns() - counters[6];
      __threadfence_system();
      for (int k = 0; k < world; ++k)
        st_release_sys(reinterpret_cast<unsigned*>(p.base[k] + off_flags) + kFlagOut + block * kPeerMaxWorld + rank, value);
    }
  }
}

}  // namespace

PeerLayout peer_layout(long long n_critic, long long n_actor, int world) {
  PeerLayout l;
  const long long q = 4ll * world;
  l.padded[kPeerCritic] = (n_critic + q - 1) / q * q;
  l.padded[kPeerActor] = (n_actor + q - 1) / q * q;
  size_t off = 4096;
  l.off_flags = 0;
  for (int b = 0; b < 2; ++b) { l.off_grads[b] = off; off += sizeof(float) * (size_t)l.padded[b]; off = (off + 255) / 256 * 256; }
  for (int b = 0; b < 2; ++b) { l.off_sums[b] = off; off += sizeof(float) * (size_t)l.padded[b]; off = (off + 255) / 256 * 256; }
  l.bytes = off;
  return l;
}

int peer_signal(PeerExchange& x, int block, cudaStream_t stream) {
  R2D2_REQUIRE(block == 0 || block == 1, "peer block");
  R2D2_REQUIRE(!x.reduce_pending[block] && !x.wait_pending[block], "peer_signal: the previous exchange of this block is not complete");
  x.epoch[block] += 1;
  peer_signal_kernel<<<1, 32, 0, stream>>>(x.ptrs, x.world, x.rank,
                                           x.lay.off_flags + sizeof(unsigned) * (kFlagIn + block * kPeerMaxWorld), x.epoch[block]);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  x.reduce_pending[block] = x.wait_pending[block] = true;
  return R2D2_OK;
}

int peer_reduce(PeerExchange& x, int block, cudaStream_t stream) {
  if (!x.reduce_pending[block]) return R2D2_OK;
  const long long slice_vec = x.lay.padded[block] / 4 / x.world;
  int grid = (int)((slice_vec + 511) / 512);
  if (grid > num_sms()) grid = num_sms();
  if (grid < 1) grid = 1;
  peer_reduce_kernel<<<grid, 512, 0, stream>>>(x.ptrs, x.world, x.rank, x.lay.off_flags, block, x.lay.off_grads[block],
                                              x.lay.off_sums[block], slice_vec, x.epoch[block]);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  x.reduce_pending[block] = false;
  return R2D2_OK;
}

int peer_wait(PeerExchange& x, int block, cudaStream_t stream) {
  R2D2_TRY(peer_reduce(x, block, stream));
  if (!x.wait_pending[block]) return R2D2_OK;
  unsigned* flags = reinterpret_cast<unsigned*>(x.ptrs.base[x.rank] + x.lay.off_flags);
  peer_wait_kernel<<<1, 32, 0, stream>>>(flags + kFlagOut + block * kPeerMaxWorld, x.world, x.epoch[block], flags + kFlagStatus,
                                         reinterpret_cast<unsigned long long*>(x.ptrs.base[x.rank] + x.lay.off_flags + kCounterBytes) + 4 + block);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  x.wait_pending[block] = false;
  return R2D2_OK;
}

int peer_status(const PeerExchange& x, int* out, cudaStream_t stream) {
  unsigned v = 0;
  R2D2_CUDA_TRY(cudaMemcpyAsync(&v, x.ptrs.base[x.rank] + x.lay.off_flags + sizeof(unsigned) * kFlagStatus, sizeof(unsigned),
                                cudaMemcpyDeviceToHost, stream));
  R2D2_CUDA_TRY(cudaStreamSynchronize(stream));
  *out = (int)v;
  return R2D2_OK;
}

int peer_counters(const PeerExchange& x, unsigned long long* out6, int reset, cudaStream_t stream) {
  char* c = x.ptrs.base[x.rank] + x.lay.off_flags + kCounterBytes;
  R2D2_CUDA_TRY(cudaMemcpyAsync(out6, c, 6 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, stream));
  if (reset) R2D2_CUDA_TRY(cudaMemsetAsync(c, 0, 6 * sizeof(unsigned long long), stream));
  R2D2_CUDA_TRY(cudaStreamSynchronize(stream));
  return R2D2_OK;
}

}  // namespace r2d2

// Exchange kernels of global sampling over the data-parallel replay shards - see replay.cuh (GlobalLayout) and
// replay.cu (replay_global_write_back / replay_global_draw).  Every kernel runs in the learner's stream; a flag is an
// iteration number stored with release semantics into the peer's exchange block after the data it covers, and read
// with acquire semantics by a bounded wait (peer_sync.cuh) whose expiry sets the block's status word.
#include "peer_sync.cuh"
#include "replay.cuh"

namespace r2d2 {

namespace {

// one CTA per destination rank k: this rank's B records go to global indices rank*B .. rank*B+B-1 of k's record block
__global__ void __launch_bounds__(256) publish_records_kernel(GlobalPeers p, GlobalLayout lay, int rank, int B,
                                                              const long long* __restrict__ leaf,
                                                              const int* __restrict__ shard,
                                                              const float* __restrict__ prio, unsigned epoch) {
  char* d = p.base[blockIdx.x];
  const size_t j0 = (size_t)rank * B;
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    reinterpret_cast<long long*>(d + lay.off_rec_leaf)[j0 + b] = leaf[b];
    reinterpret_cast<int*>(d + lay.off_rec_shard)[j0 + b] = shard[b];
    reinterpret_cast<float*>(d + lay.off_rec_prio)[j0 + b] = prio[b];
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) st_release_sys(reinterpret_cast<unsigned*>(d) + kGlobalFlagPub + rank, epoch);
}

// one CTA per destination rank k: this shard's root into k's totals[rank], this rank's uniforms into k's uniforms
__global__ void __launch_bounds__(256) publish_root_kernel(GlobalPeers p, GlobalLayout lay, int rank, int B,
                                                           const float* __restrict__ root, const float* __restrict__ u,
                                                           unsigned epoch) {
  char* d = p.base[blockIdx.x];
  for (int b = threadIdx.x; b < B; b += blockDim.x)
    reinterpret_cast<float*>(d + lay.off_uniforms)[(size_t)rank * B + b] = u[b];
  if (threadIdx.x == 0) reinterpret_cast<float*>(d + kGlobalOffTotals)[rank] = *root;
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) st_release_sys(reinterpret_cast<unsigned*>(d) + kGlobalFlagTot + rank, epoch);
}

// after the gather: "my rows of the next batch are in your slot", with this owner's minimum drawn leaf
__global__ void global_deliver_kernel(GlobalPeers p, int world, int rank, unsigned epoch) {
  const int k = threadIdx.x;
  if (k < world) {
    __threadfence_system();   // the draw and gather kernels ahead of this one in the stream happen-before the flag
    const float m = *reinterpret_cast<const float*>(p.base[rank] + kGlobalOffOwnMin);
    reinterpret_cast<float*>(p.base[k] + kGlobalOffMinima)[rank] = m;
    st_release_sys(reinterpret_cast<unsigned*>(p.base[k]) + kGlobalFlagDel + rank, epoch);
  }
}

// Single CTA on the consumer: wait for every owner's delivery, then w[b] = (min_global / leaf_b)^beta with
// min_global = min over the owners' minima - the same min and the same formula as is_weight_kernel over the
// concatenated W*B batch (fminf is exact and order-free), so the weights equal it bit for bit.
__global__ void __launch_bounds__(256) global_receive_kernel(GlobalPeers p, GlobalLayout lay, int world, int rank, int B,
                                                             int slot, int weighted, float beta, unsigned epoch) {
  char* own = p.base[rank];
  unsigned* flags = reinterpret_cast<unsigned*>(own);
  if ((int)threadIdx.x < world) spin_until(flags + kGlobalFlagDel + threadIdx.x, epoch, flags + kGlobalStatus);
  __syncthreads();
  if (!weighted) return;
  const volatile float* minima = reinterpret_cast<const volatile float*>(own + kGlobalOffMinima);
  float m = INFINITY;
  for (int k = 0; k < world; ++k) m = fminf(m, minima[k]);
  volatile float* w = reinterpret_cast<volatile float*>(own + lay.slot(slot) + lay.off_weight);
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    const float leaf = w[b];
    w[b] = (beta == 0.f || !(leaf > 0.f)) ? 1.0f : powf(__fdiv_rn(m, leaf), beta);
  }
}

}  // namespace

int global_publish_records(const GlobalPeers& p, const GlobalLayout& lay, int world, int rank, int B,
                           const long long* leaf, const int* shard, const float* prio, unsigned epoch, cudaStream_t st) {
  publish_records_kernel<<<world, 256, 0, st>>>(p, lay, rank, B, leaf, shard, prio, epoch);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

int global_publish_root(const GlobalPeers& p, const GlobalLayout& lay, int world, int rank, int B, int slot,
                        const float* root, unsigned epoch, cudaStream_t st) {
  const float* u = reinterpret_cast<const float*>(p.base[rank] + lay.slot(slot) + lay.off_slot_uniforms);
  publish_root_kernel<<<world, 256, 0, st>>>(p, lay, rank, B, root, u, epoch);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

int global_deliver(const GlobalPeers& p, int world, int rank, unsigned epoch, cudaStream_t st) {
  global_deliver_kernel<<<1, 32, 0, st>>>(p, world, rank, epoch);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

int global_receive(const GlobalPeers& p, const GlobalLayout& lay, int world, int rank, int B, int slot, bool weighted,
                   float beta, unsigned epoch, cudaStream_t st) {
  global_receive_kernel<<<1, 256, 0, st>>>(p, lay, world, rank, B, slot, weighted ? 1 : 0, beta, epoch);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

}  // namespace r2d2

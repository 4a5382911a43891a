// gemm_f32 on the Hopper tensor cores (sm_90a, wgmma):
//
//  1. operand images: every operand is bf16 hi/lo planes stored TILE-MAJOR in exactly the shared-memory image the MMA
//     wants - one 16 KB block per (128-row tile, 32-deep k tile) = hi plane (8 KB) + lo plane (8 KB) in core-matrix
//     order (no swizzle), zero padded.  Producers that can write it directly do (GemmParams::A_img / B_img, the l1
//     kernel for z1); otherwise pack_operand_kernel converts the fp32 tensor (any leading dimension, ragged edges) in an
//     HBM-bound elementwise pass (8 B/element).
//  2. gemm_packed_kernel: per CTA one 128 x 128 output tile, two CTAs per SM.  A producer thread streams the tile images
//     with 1-D bulk copies (cp.async.bulk ... mbarrier::complete_tx, no tensor map, no per-element work) through a
//     3-stage ring; two consumer warpgroups each issue wgmma.m64n128k16 (passes lo*hi + hi*lo + hi*hi) into register
//     accumulators, keeping one k tile of wgmma in flight while they wait for the next, and apply bias / tanh / dtanh /
//     +Z or the split-K reduction straight from the accumulator fragments.
//
// Why images instead of fp32 operands: the image is the same byte count as the fp32 operand, is re-read ~N/128 (A)
// or ~M/128 (B) times from L2, and needs no conversion inside the GEMM's main loop.
#include <stdlib.h>

#include <map>
#include <mutex>
#include <utility>

#include "elementwise.cuh"
#include "gemm.cuh"
#include "sm90.cuh"

namespace r2d2 {
namespace {

constexpr int TBM = 128, TBN = 128, TBK = 32;
constexpr int PLANE_BYTES = 128 * TBK * 2;     // 8 KB: one bf16 plane of a 128 x 32 operand tile
constexpr int TILE_BYTES = 2 * PLANE_BYTES;    // 16 KB: hi plane + lo plane of one operand tile
constexpr int PACKED_GEMM_THREADS = 288;       // warpgroups 0..1 wgmma + epilogue, warp 8 producer
// two CTAs per SM (2 x 96 KB ring, 2 x 288 threads x 96 registers): one CTA's ring fill and epilogue run while the
// other's wgmmas keep the tensor pipe busy
constexpr int CTAS_PER_SM = 2;
constexpr int STAGES = 3;
constexpr int STAGE_BYTES = 2 * TILE_BYTES;    // A tile + B tile
constexpr int OFF_BARS = STAGES * STAGE_BYTES;
constexpr int PACKED_SMEM = OFF_BARS + 128;

// ---- operand tile image (shared with the MMA descriptors below) --------------------------------------------------
// a tile is 512 groups of 8 elements; group `id` lives at byte id*16 of each plane.
//   K-major  (source [row][k], k contiguous):  row = 8*(id/32) + id%8, k = 8*((id/8)%4) ..   [row/8][k/8][row%8][16 B]
//                                              descriptor LBO (k-group stride) = 128, SBO (8-row-group stride) = 512
//   MN-major (source [k][mn], mn contiguous):  k = 8*(id/128) + id%8, mn = 8*((id/8)%16) ..  [k/8][mn/8][k%8][16 B]
//                                              descriptor LBO (k-group stride) = 2048, SBO (8-mn-group stride) = 128
template <bool MN_MAJOR>
__global__ void __launch_bounds__(256) pack_operand_kernel(const float* __restrict__ src, long long ld, int mn_lim,
                                                           int k_lim, int k_tiles_total, int k_tile_offset, int vec,
                                                           unsigned char* __restrict__ dst) {
  const int mn0 = blockIdx.y * 128, k0 = blockIdx.x * TBK;
  unsigned char* tile = dst + ((size_t)blockIdx.y * k_tiles_total + k_tile_offset + blockIdx.x) * TILE_BYTES;
#pragma unroll
  for (int g = 0; g < 2; ++g) {
    const int id = threadIdx.x + g * 256;
    int row, col, row_lim, col_lim;
    if (MN_MAJOR) { row = k0 + 8 * (id >> 7) + (id & 7); col = mn0 + 8 * ((id >> 3) & 15); row_lim = k_lim; col_lim = mn_lim; }
    else          { row = mn0 + 8 * (id >> 5) + (id & 7); col = k0 + 8 * ((id >> 3) & 3);  row_lim = mn_lim; col_lim = k_lim; }
    float v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = 0.f;
    if (row < row_lim && col < col_lim) {
      const float* p = src + (long long)row * ld + col;
      if (vec && col + 7 < col_lim) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p + 4));
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) if (col + i < col_lim) v[i] = __ldg(p + i);
      }
    }
    uint4 h, l;
    split_pack2(v[0], v[1], h.x, l.x);
    split_pack2(v[2], v[3], h.y, l.y);
    split_pack2(v[4], v[5], h.z, l.z);
    split_pack2(v[6], v[7], h.w, l.w);
    *reinterpret_cast<uint4*>(tile + id * 16) = h;
    *reinterpret_cast<uint4*>(tile + PLANE_BYTES + id * 16) = l;
  }
}

__device__ __forceinline__ void mbar_wait_spin(uint64_t* bar, uint32_t parity) {
  while (!sm90::mbar_try_wait(bar, parity)) {}
}

struct PackedGemmParams {
  const unsigned char* pa;   // [m_tiles][k_tiles][16 KB]
  const unsigned char* pb;   // [n_tiles][k_tiles][16 KB]
  int k_tiles;
  float* C; long long ldc;
  int M, N;
  const float* bias;
  const float* bias2;
  const float* Z; long long ldz;
  int epilogue, split_k;
  long long c_split_stride;  // split_k > 1: CTA z writes its partial product to C + z * c_split_stride
  unsigned char* c_img_k;    // optional: C also leaves as packed operand images (N % 32 == 0, split_k == 1), see epilogue
  unsigned char* c_img_mn;
};

// warpgroups 0 and 1 = consumers, each owning 64 rows of the 128 x 128 output tile as wgmma register accumulators;
// warp 8 = producer (one elected thread).
template <bool A_MN, bool B_MN>
__global__ void __launch_bounds__(PACKED_GEMM_THREADS, CTAS_PER_SM) gemm_packed_kernel(PackedGemmParams p) {
  extern __shared__ __align__(128) unsigned char smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + OFF_BARS);   // [STAGES] bytes landed
  uint64_t* empty = full + STAGES;                                  // [STAGES] both consumer warpgroups done reading

  const int tid = threadIdx.x, lane = tid & 31;
  const int wg = __shfl_sync(0xffffffffu, tid >> 7, 0);
  const int m_tile = blockIdx.y, n_tile = blockIdx.x;
  const int m0 = m_tile * TBM, n0 = n_tile * TBN;
  const int per_split = (p.k_tiles + p.split_k - 1) / p.split_k;
  const int t_begin = blockIdx.z * per_split;
  const int t_end = min(p.k_tiles, t_begin + per_split);
  if (t_begin >= t_end) return;
  const int n_tiles = t_end - t_begin;

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) { sm90::mbar_init(&full[s], 1); sm90::mbar_init(&empty[s], 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wg == 2) {
    // ================= producer: one 16 KB bulk copy per operand tile and k tile =================
    if (sm90::elect_one()) {
      const unsigned char* a_src = p.pa + ((size_t)m_tile * p.k_tiles + t_begin) * TILE_BYTES;
      const unsigned char* b_src = p.pb + ((size_t)n_tile * p.k_tiles + t_begin) * TILE_BYTES;
      const uint32_t smem_base = sm90::smem_u32(smem);
      for (int i = 0; i < n_tiles; ++i) {
        const int s = i % STAGES;
        mbar_wait_spin(&empty[s], ((i / STAGES) & 1) ^ 1);
        const uint32_t bar = sm90::smem_u32(&full[s]);
        sm90::mbar_arrive_expect_tx(&full[s], 2 * TILE_BYTES);
        sm90::bulk_copy_g2s(smem_base + s * STAGE_BYTES, a_src + (size_t)i * TILE_BYTES, TILE_BYTES, bar);
        sm90::bulk_copy_g2s(smem_base + s * STAGE_BYTES + TILE_BYTES, b_src + (size_t)i * TILE_BYTES, TILE_BYTES, bar);
      }
    }
    return;
  }

  // ================= consumers: rows [64 wg, 64 wg + 64) of the tile =================
  const int half = wg, t = tid & 127;
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  // tile image layouts (top of this file): K-major LBO 128 / SBO 512, MN-major LBO 2048 / SBO 128
  const uint32_t a_lbo = A_MN ? 2048 : 128, a_sbo = A_MN ? 128 : 512;
  const uint32_t b_lbo = B_MN ? 2048 : 128, b_sbo = B_MN ? 128 : 512;
  const uint32_t a_ks = A_MN ? 4096 : 256, b_ks = B_MN ? 4096 : 256;     // byte advance per K=16 step
  const uint32_t a_half = half * 8 * a_sbo;                               // 64 rows = eight 8-row groups
  const uint32_t smem_base = sm90::smem_u32(smem);
  for (int i = 0; i < n_tiles; ++i) {
    const int s = i % STAGES;
    mbar_wait_spin(&full[s], (i / STAGES) & 1);
    const uint32_t sa = smem_base + s * STAGE_BYTES + a_half, sb = smem_base + s * STAGE_BYTES + TILE_BYTES;
    sm90::fence_regs(acc);
    sm90::wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < TBK / 16; ++ks) {
      const uint64_t a_hi = sm90::make_smem_desc(sa + ks * a_ks, a_lbo, a_sbo);
      const uint64_t a_lo = sm90::make_smem_desc(sa + ks * a_ks + PLANE_BYTES, a_lbo, a_sbo);
      const uint64_t b_hi = sm90::make_smem_desc(sb + ks * b_ks, b_lbo, b_sbo);
      const uint64_t b_lo = sm90::make_smem_desc(sb + ks * b_ks + PLANE_BYTES, b_lbo, b_sbo);
      sm90::wgmma_m64n128k16_bf16<A_MN, B_MN>(acc, a_lo, b_hi);
      sm90::wgmma_m64n128k16_bf16<A_MN, B_MN>(acc, a_hi, b_lo);
      sm90::wgmma_m64n128k16_bf16<A_MN, B_MN>(acc, a_hi, b_hi);
    }
    sm90::wgmma_commit();
    sm90::wgmma_wait<1>();   // k tile i - 1 is done, k tile i stays in flight
    sm90::fence_regs(acc);
    __syncwarp();
    if (i > 0 && t == 0) sm90::mbar_arrive(&empty[(i - 1) % STAGES]);
  }
  sm90::wgmma_wait<0>();
  sm90::fence_regs(acc);
  __syncwarp();
  if (t == 0) sm90::mbar_arrive(&empty[(n_tiles - 1) % STAGES]);

  // ================= epilogue straight from the accumulator fragments =================
  // fragment j of a thread: rows r and r + 8, columns c, c + 1 with r = 16 (t / 32) + (t % 32) / 4, c = 8 j + 2 (t % 4)
  const int r_base = m0 + half * 64 + 16 * (t >> 5) + (lane >> 2);
  const int c_off = 2 * (lane & 3);
  float* const C = p.C + (long long)blockIdx.z * p.c_split_stride;
  const bool vec_c = ((reinterpret_cast<uintptr_t>(C) & 7) == 0) && (p.ldc % 2 == 0);
  const bool img = p.c_img_k != nullptr || p.c_img_mn != nullptr;   // kernel-uniform
#pragma unroll
  for (int j = 0; j < TBN / 8; ++j) {
    const int col = n0 + 8 * j + c_off;
    const bool c0ok = col < p.N, c1ok = col + 1 < p.N;
    float b0 = 0.f, b1 = 0.f;
    if (p.bias) {
      if (c0ok) b0 = __ldg(p.bias + col) + (p.bias2 ? __ldg(p.bias2 + col) : 0.f);
      if (c1ok) b1 = __ldg(p.bias + col + 1) + (p.bias2 ? __ldg(p.bias2 + col + 1) : 0.f);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = r_base + 8 * h;
      float v0 = acc[4 * j + 2 * h] + b0, v1 = acc[4 * j + 2 * h + 1] + b1;
      if (img) {
        // C also leaves as the bf16 hi/lo operand image(s) of the product(s) that consume it next: a 16-byte piece = 8
        // consecutive columns of one row, held by the 4 lanes of a quad.  Every lane takes part in the shuffles; rows
        // >= M are written as zeros (a reduction index in the MN-major image).
        const bool ok = row < p.M && c0ok;
        if (ok) {
          if (p.epilogue == EPI_TANH) { v0 = tanhf(v0); v1 = tanhf(v1); }
          *reinterpret_cast<float2*>(p.C + (long long)row * p.ldc + col) = make_float2(v0, v1);   // N % 32 == 0
        } else {
          v0 = v1 = 0.f;
        }
        uint32_t hw, lw;
        split_pack2(v0, v1, hw, lw);
        const int q0 = lane & ~3;
        const uint4 hi = make_uint4(__shfl_sync(0xffffffffu, hw, q0), __shfl_sync(0xffffffffu, hw, q0 + 1),
                                    __shfl_sync(0xffffffffu, hw, q0 + 2), __shfl_sync(0xffffffffu, hw, q0 + 3));
        const uint4 lo = make_uint4(__shfl_sync(0xffffffffu, lw, q0), __shfl_sync(0xffffffffu, lw, q0 + 1),
                                    __shfl_sync(0xffffffffu, lw, q0 + 2), __shfl_sync(0xffffffffu, lw, q0 + 3));
        const int cg = n0 + 8 * j;   // first column of the 16-byte piece
        if ((lane & 3) == 0 && cg < p.N && row < ((p.M + 31) & ~31)) {
          if (p.c_img_k && row < p.M) {
            unsigned char* d = p.c_img_k + ((size_t)(row >> 7) * (p.N >> 5) + (cg >> 5)) * TILE_BYTES +
                               ((((row & 127) >> 3) * 32) + ((cg & 31) >> 3) * 8 + (row & 7)) * 16;
            *reinterpret_cast<uint4*>(d) = hi;
            *reinterpret_cast<uint4*>(d + PLANE_BYTES) = lo;
          }
          if (p.c_img_mn) {
            unsigned char* d = p.c_img_mn + ((size_t)(cg >> 7) * ((p.M + 31) >> 5) + (row >> 5)) * TILE_BYTES +
                               ((((row & 31) >> 3) * 128) + ((cg & 127) >> 3) * 8 + (row & 7)) * 16;
            *reinterpret_cast<uint4*>(d) = hi;
            *reinterpret_cast<uint4*>(d + PLANE_BYTES) = lo;
          }
        }
        continue;
      }
      if (row >= p.M || !c0ok) continue;
      if (p.epilogue == EPI_TANH) {
        v0 = tanhf(v0); v1 = tanhf(v1);
      } else if (p.epilogue == EPI_MUL_DTANH || p.epilogue == EPI_ADD_Z) {
        const float* z = p.Z + (long long)row * p.ldz + col;
        const float z0 = z[0], z1 = c1ok ? z[1] : 0.f;
        if (p.epilogue == EPI_MUL_DTANH) { v0 *= 1.f - z0 * z0; v1 *= 1.f - z1 * z1; }
        else { v0 += z0; v1 += z1; }
      }
      float* cp = C + (long long)row * p.ldc + col;
      if (vec_c && c1ok) {
        *reinterpret_cast<float2*>(cp) = make_float2(v0, v1);
      } else {
        cp[0] = v0;
        if (c1ok) cp[1] = v1;
      }
    }
  }
}

// grow-only scratch for the packed operand images, one set per (device, stream): kernels of one stream are ordered,
// so a pack pass and the GEMM that reads it never overlap with the next call's pack on the same buffers; different
// streams (other learners, other devices, other host threads) never share a buffer.
struct Scratch { unsigned char* ptr = nullptr; size_t bytes = 0; };
struct LastPackedA { const float* ptr = nullptr; long long ld = 0; int mn = 0, k = 0, mn_major = 0, k_tiles = 0; };
struct StreamScratch { Scratch a, b; LastPackedA last_a; };
std::mutex g_scratch_mutex;
std::map<std::pair<int, cudaStream_t>, StreamScratch> g_scratch;

int scratch_for(cudaStream_t stream, StreamScratch** out) {
  int dev = 0;
  R2D2_CUDA_TRY(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(g_scratch_mutex);
  *out = &g_scratch[std::make_pair(dev, stream)];   // std::map: references stay valid across insertions
  return R2D2_OK;
}

int ensure_scratch(Scratch& s, size_t bytes) {
  if (s.bytes >= bytes) return R2D2_OK;
  if (s.ptr) { R2D2_CUDA_TRY(cudaDeviceSynchronize()); R2D2_CUDA_TRY(cudaFree(s.ptr)); s.ptr = nullptr; s.bytes = 0; }
  const size_t want = bytes + bytes / 4 + (1u << 20);
  R2D2_CUDA_TRY(cudaMalloc(&s.ptr, want));
  s.bytes = want;
  return R2D2_OK;
}

int launch_pack(const float* src, long long ld, int mn_lim, int k_lim, bool mn_major, int mn_tiles, int k_tiles_total,
                int k_tile_offset, unsigned char* dst, cudaStream_t stream) {
  const int vec = (((reinterpret_cast<uintptr_t>(src) & 15) == 0) && (ld % 4 == 0)) ? 1 : 0;
  dim3 grid(ceil_div(k_lim, TBK), mn_tiles);
  if (mn_major) pack_operand_kernel<true><<<grid, 256, 0, stream>>>(src, ld, mn_lim, k_lim, k_tiles_total, k_tile_offset, vec, dst);
  else          pack_operand_kernel<false><<<grid, 256, 0, stream>>>(src, ld, mn_lim, k_lim, k_tiles_total, k_tile_offset, vec, dst);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

}  // namespace

int gemm_tc_suggest_split_k(int M, int N, int K) {
  long long tiles = (long long)ceil_div(M, TBM) * ceil_div(N, TBN);
  int k_tiles = ceil_div(K, TBK);
  if (tiles >= num_sms() || k_tiles < 16) return 1;
  int want = (int)ceil_div_ll(2 * num_sms(), tiles);
  int max_by_k = k_tiles / 8;
  int s = want < max_by_k ? want : max_by_k;
  if (s < 1) s = 1;
  if (s > 256) s = 256;
  return s;
}

template <bool A_MN, bool B_MN>
int launch_packed(const PackedGemmParams& q, int m_tiles, int n_tiles, int slices, cudaStream_t stream) {
  static PerDeviceOnce once;
  if (once.need()) {
    R2D2_CUDA_TRY(cudaFuncSetAttribute(gemm_packed_kernel<A_MN, B_MN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       PACKED_SMEM));
  }
  dim3 grid(n_tiles, m_tiles, slices);
  gemm_packed_kernel<A_MN, B_MN><<<grid, PACKED_GEMM_THREADS, PACKED_SMEM, stream>>>(q);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

int gemm_f32_tc(const GemmParams& p, GemmLayout layout, cudaStream_t stream) {
  const bool a_mn = (layout == GEMM_TN), b_mn = (layout != GEMM_NT);
  const int m_tiles = ceil_div(p.M, TBM), n_tiles = ceil_div(p.N, TBN);
  const int kt1 = ceil_div(p.K, TBK), kt2 = p.K2 > 0 ? ceil_div(p.K2, TBK) : 0;
  const int k_tiles = kt1 + kt2;
  R2D2_REQUIRE(m_tiles <= 65535, "M too large for grid.y");
  StreamScratch* sc = nullptr;
  R2D2_TRY(scratch_for(stream, &sc));
  Scratch& g_pack_a = sc->a;
  Scratch& g_pack_b = sc->b;
  LastPackedA& last_a = sc->last_a;
  if (!p.A_img) R2D2_TRY(ensure_scratch(g_pack_a, (size_t)m_tiles * k_tiles * TILE_BYTES));
  if (!p.B_img) R2D2_TRY(ensure_scratch(g_pack_b, (size_t)n_tiles * k_tiles * TILE_BYTES));
  // key of the image currently held in the A scratch: reuse is honoured only if the caller asks AND the key matches
  const bool reuse = p.reuse_packed_a && kt2 == 0 && last_a.ptr == p.A && last_a.ld == p.lda && last_a.mn == p.M &&
                     last_a.k == p.K && last_a.mn_major == (a_mn ? 1 : 0) && last_a.k_tiles == k_tiles;
  if (!p.A_img) {
    if (!reuse) R2D2_TRY(launch_pack(p.A, p.lda, p.M, p.K, a_mn, m_tiles, k_tiles, 0, g_pack_a.ptr, stream));
    last_a = LastPackedA{kt2 ? nullptr : p.A, p.lda, p.M, p.K, a_mn ? 1 : 0, k_tiles};
  }
  if (!p.B_img) R2D2_TRY(launch_pack(p.B, p.ldb, p.N, p.K, b_mn, n_tiles, k_tiles, 0, g_pack_b.ptr, stream));
  if (kt2) {
    R2D2_REQUIRE(!p.A_img && !p.B_img, "packed operand with a second K segment");
    R2D2_TRY(launch_pack(p.A2, p.lda2, p.M, p.K2, a_mn, m_tiles, k_tiles, kt1, g_pack_a.ptr, stream));
    R2D2_TRY(launch_pack(p.B2, p.ldb2, p.N, p.K2, b_mn, n_tiles, k_tiles, kt1, g_pack_b.ptr, stream));
  }
  PackedGemmParams q;
  q.pa = p.A_img ? p.A_img : g_pack_a.ptr; q.pb = p.B_img ? p.B_img : g_pack_b.ptr; q.k_tiles = k_tiles; q.C = p.C; q.ldc = p.ldc; q.M = p.M; q.N = p.N;
  q.bias = p.bias; q.bias2 = p.bias ? p.bias2 : nullptr; q.Z = p.Z; q.ldz = p.ldz; q.epilogue = p.epilogue; q.split_k = p.split_k;
  q.c_img_k = p.C_img_k; q.c_img_mn = p.C_img_mn;
  q.c_split_stride = 0;
  int slices = 1;
  if (p.split_k > 1) {   // partial products into slices, then added into C in slice order (same bits every run)
    slices = ceil_div(k_tiles, ceil_div(k_tiles, p.split_k));   // every slice z < slices owns at least one k tile
    R2D2_TRY(partials_scratch((size_t)slices * p.M * p.N, stream, &q.C));
    q.ldc = p.N;
    q.c_split_stride = (long long)p.M * p.N;
  }
  if (p.C_img_k || p.C_img_mn) {
    R2D2_REQUIRE(p.N % 32 == 0 && p.split_k == 1 && (p.epilogue == EPI_NONE || p.epilogue == EPI_TANH) &&
                     (reinterpret_cast<uintptr_t>(p.C) & 7) == 0 && p.ldc % 2 == 0,
                 "operand image from the wgmma epilogue: N % 32 == 0, no split-K, bias / tanh epilogue, 8-byte aligned C");
  }
  if (a_mn) R2D2_TRY((launch_packed<true, true>(q, m_tiles, n_tiles, slices, stream)));      // TN
  else if (b_mn) R2D2_TRY((launch_packed<false, true>(q, m_tiles, n_tiles, slices, stream)));   // NN
  else R2D2_TRY((launch_packed<false, false>(q, m_tiles, n_tiles, slices, stream)));          // NT
  if (p.split_k > 1) return add_partials(q.C, slices, p.M, p.N, p.C, p.ldc, nullptr, stream);
  return R2D2_OK;
}

}  // namespace r2d2

// Degenerate contractions of the learner path as plain fp32 FMA kernels.
//
// A third of the GEMM launches of one iteration have a dimension of 6..23 (obs / action widths, models.py:17-19,
// :62-64): x*W1^T (K = 17 | 17+6), the heads (N = 6), their dgrads and the dW1 / dW3 blocks.  On a 128-wide tensor
// core tile they are >90% padding although they only stream 2-32 MB.  Here every one is a single HBM-bound pass in
// exact fp32:
//   thin_smallk : C[M,N] = epi(A[M,K] W (+ A2[M,K2] W2) + bias),  K + K2 <= 32   (NT / NN)
//   thin_smalln : C[M,N] = epi(A[M,K] W + bias),                  N <= 32        (NT / NN)
//   thin_tn     : C[M,N] += A[K,M]^T B[K,N],                      M <= 32 or N <= 32, reduction over K rows
#include "elementwise.cuh"
#include "gemm.cuh"
#include "sm90.cuh"

namespace r2d2 {
namespace {

__device__ __forceinline__ float apply_epilogue(float v, int epilogue, float z) {
  if (epilogue == EPI_TANH) return sm90::tanh_fast(v);
  if (epilogue == EPI_MUL_DTANH) return v * (1.f - z * z);
  if (epilogue == EPI_ADD_Z) return v + z;
  return v;
}

// ------------------------------------------------------------------------------------------------
// small K.  Block = 256 threads = 32 rows x 256 columns per pass (thread: 8 rows x 4 columns).  W stays in shared
// memory for the whole (persistent) block; the A rows of the next pass arrive by cp.async while this pass computes.
// ------------------------------------------------------------------------------------------------
constexpr int SK_ROWS = 32, SK_COLS = 256, SK_KMAX = 32, SK_THREADS = 256, SK_WLD = SK_COLS + 4;

using sm90::cp_async_4;
using sm90::cp_async_commit;
using sm90::cp_async_wait_all;

template <bool NN>
__global__ void __launch_bounds__(SK_THREADS) thin_smallk_kernel(GemmParams p, int vec_c, int vec_z) {
  __shared__ __align__(16) float Ws[SK_KMAX][SK_WLD];        // row stride 260: transposed fill is 4-way, not 32-way, conflicted
  __shared__ __align__(16) float As[2][SK_ROWS][SK_KMAX];
  const int tid = threadIdx.x;
  const int n0 = blockIdx.y * SK_COLS;
  const int Kt = p.K + p.K2;
  for (int idx = tid; idx < SK_KMAX * SK_WLD; idx += SK_THREADS) (&Ws[0][0])[idx] = 0.f;
  for (int idx = tid; idx < 2 * SK_ROWS * SK_KMAX; idx += SK_THREADS) (&As[0][0][0])[idx] = 0.f;
  __syncthreads();
  {   // thread = column tid of the tile; the (<= 32) loads of a batch are all in flight before the first store
    const int n = n0 + tid;
    for (int kb = 0; kb < Kt; kb += 8) {
      float wv[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int k = kb + i;
        wv[i] = 0.f;
        if (n < p.N && k < Kt) {
          if (NN) wv[i] = __ldg(p.B + (long long)k * p.ldb + n);
          else    wv[i] = (k < p.K) ? __ldg(p.B + (long long)n * p.ldb + k) : __ldg(p.B2 + (long long)n * p.ldb2 + (k - p.K));
        }
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) if (kb + i < SK_KMAX) Ws[kb + i][tid] = wv[i];
    }
  }
  const int cg = tid & 63, rgp = tid >> 6;
  const int col = n0 + cg * 4;
  float bias[4] = {0.f, 0.f, 0.f, 0.f};
  if (p.bias) {
#pragma unroll
    for (int j = 0; j < 4; ++j) if (col + j < p.N) bias[j] = __ldg(p.bias + col + j);
  }
  const int k4n = (Kt + 3) >> 2;
  const int row_tiles = (p.M + SK_ROWS - 1) / SK_ROWS;
  auto stage = [&](int rt, int buf) {   // rows past M keep the zeros of the initial fill or of an earlier tile: never stored
    const int r = tid >> 3, row = rt * SK_ROWS + r;
    if (row < p.M) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int k = (tid & 7) + 8 * j;
        if (k < Kt) cp_async_4(&As[buf][r][k], (k < p.K) ? p.A + (long long)row * p.lda + k : p.A2 + (long long)row * p.lda2 + (k - p.K));
      }
    }
    cp_async_commit();
  };
  int it = 0;
  if ((int)blockIdx.x < row_tiles) stage(blockIdx.x, 0);
  cp_async_wait_all();
  __syncthreads();
  const bool needs_z = p.epilogue == EPI_MUL_DTANH || p.epilogue == EPI_ADD_Z;
  for (int rt = blockIdx.x; rt < row_tiles; rt += gridDim.x, ++it) {
    const int buf = it & 1;
    const int r0 = rt * SK_ROWS;
    if (rt + (int)gridDim.x < row_tiles) stage(rt + gridDim.x, buf ^ 1);
    float acc[8][4];
#pragma unroll
    for (int r = 0; r < 8; ++r)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[r][j] = bias[j];
    for (int k4 = 0; k4 < k4n; ++k4) {
      const float4 w0 = *reinterpret_cast<const float4*>(&Ws[4 * k4 + 0][cg * 4]);
      const float4 w1 = *reinterpret_cast<const float4*>(&Ws[4 * k4 + 1][cg * 4]);
      const float4 w2 = *reinterpret_cast<const float4*>(&Ws[4 * k4 + 2][cg * 4]);
      const float4 w3 = *reinterpret_cast<const float4*>(&Ws[4 * k4 + 3][cg * 4]);
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const float4 a = *reinterpret_cast<const float4*>(&As[buf][rgp * 8 + r][4 * k4]);
        acc[r][0] = fmaf(a.w, w3.x, fmaf(a.z, w2.x, fmaf(a.y, w1.x, fmaf(a.x, w0.x, acc[r][0]))));
        acc[r][1] = fmaf(a.w, w3.y, fmaf(a.z, w2.y, fmaf(a.y, w1.y, fmaf(a.x, w0.y, acc[r][1]))));
        acc[r][2] = fmaf(a.w, w3.z, fmaf(a.z, w2.z, fmaf(a.y, w1.z, fmaf(a.x, w0.z, acc[r][2]))));
        acc[r][3] = fmaf(a.w, w3.w, fmaf(a.z, w2.w, fmaf(a.y, w1.w, fmaf(a.x, w0.w, acc[r][3]))));
      }
    }
    if (col < p.N) {
      const bool full = col + 3 < p.N;
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const int row = r0 + rgp * 8 + r;
        if (row >= p.M) break;
        float z[4] = {0.f, 0.f, 0.f, 0.f};
        if (needs_z) {
          const float* zp = p.Z + (long long)row * p.ldz + col;
          if (full && vec_z) { const float4 t = *reinterpret_cast<const float4*>(zp); z[0] = t.x; z[1] = t.y; z[2] = t.z; z[3] = t.w; }
          else {
#pragma unroll
            for (int j = 0; j < 4; ++j) if (col + j < p.N) z[j] = zp[j];
          }
        }
        float v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = apply_epilogue(acc[r][j], p.epilogue, z[j]);
        float* cp = p.C + (long long)row * p.ldc + col;
        if (full && vec_c) *reinterpret_cast<float4*>(cp) = make_float4(v[0], v[1], v[2], v[3]);
        else {
#pragma unroll
          for (int j = 0; j < 4; ++j) if (col + j < p.N) cp[j] = v[j];
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[r][j] = v[j];   // keep the finished values for the image below
      }
    }
    if (p.C_img_k || p.C_img_mn) {
      // C also leaves as the K-major bf16 hi/lo operand image of the product that consumes it next (gemm_tc.cu tile
      // format, K = N of this call): lanes 2i / 2i+1 hold the two halves of an 8-column chunk, so they swap rows
      // (even lane ends with rows 0-3 x 8 columns, odd lane with rows 4-7) and write 32-byte pieces = two rows of a
      // core matrix with one 256-bit store each.
      const bool odd = (tid & 1) != 0;
      float own[4][4], oth[4][4];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float send = odd ? acc[i][j] : acc[4 + i][j];
          oth[i][j] = __shfl_xor_sync(0xffffffffu, send, 1);
          own[i][j] = odd ? acc[4 + i][j] : acc[i][j];
        }
      const int m0 = r0 + rgp * 8;
      const int c8 = col >> 3;
      if (col < p.N) {
        unsigned char* base = p.C_img_k ? p.C_img_k + ((size_t)(m0 >> 7) * (p.N >> 5) + (c8 >> 2)) * 16384 +
                                              ((((m0 & 127) >> 3) * 32) + (c8 & 3) * 8) * 16 + (odd ? 64 : 0) : nullptr;
        // MN-major twin (rows = reduction index): tile (col / 128, row / 32), same 16-byte chunks
        unsigned char* base_mn = p.C_img_mn ? p.C_img_mn + ((size_t)(c8 >> 4) * ((p.M + 31) >> 5) + (m0 >> 5)) * 16384 +
                                                  ((((m0 & 31) >> 3) * 128) + (c8 & 15) * 8) * 16 + (odd ? 64 : 0) : nullptr;
#pragma unroll
        for (int pr = 0; pr < 2; ++pr) {     // row pairs (0,1) and (2,3) of this lane's four rows
          float hi8[8], lo8[8];
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            const int i = 2 * pr + rr;
            float x[8];
#pragma unroll
            for (int j = 0; j < 4; ++j) { x[j] = odd ? oth[i][j] : own[i][j]; x[4 + j] = odd ? own[i][j] : oth[i][j]; }
            if (m0 + (odd ? 4 : 0) + i >= p.M) {   // in the MN-major image the rows are a reduction index: must read as zero
#pragma unroll
              for (int j = 0; j < 8; ++j) x[j] = 0.f;
            }
            uint32_t h[4], l[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) split_pack2(x[2 * j], x[2 * j + 1], h[j], l[j]);
#pragma unroll
            for (int j = 0; j < 4; ++j) { hi8[rr * 4 + j] = __uint_as_float(h[j]); lo8[rr * 4 + j] = __uint_as_float(l[j]); }
          }
          if (m0 + (odd ? 4 : 0) + 2 * pr < p.M) {       // rows past M only feed masked output rows of the consumer
            if (base) {
              st_global_v8(reinterpret_cast<float*>(base + pr * 32), hi8);
              st_global_v8(reinterpret_cast<float*>(base + 8192 + pr * 32), lo8);
            }
            if (base_mn) {
              st_global_v8(reinterpret_cast<float*>(base_mn + pr * 32), hi8);
              st_global_v8(reinterpret_cast<float*>(base_mn + 8192 + pr * 32), lo8);
            }
          }
        }
      }
    }
    cp_async_wait_all();
    __syncthreads();   // next tile landed; everyone is done reading this one
  }
}

// ------------------------------------------------------------------------------------------------
// small N.  One warp per group of R = 32 / NP rows; lane owns the k slices {128 j + 4 lane .. +3}; W^T[n][k] in shared
// memory.  The R*NP = 32 partial sums of a lane are reduced across the warp with a halving exchange (31 shuffles):
// afterwards lane L holds output (row L / NP, column L % NP).
// ------------------------------------------------------------------------------------------------
constexpr int SN_THREADS = 256;

template <bool NN, int NP>
__global__ void __launch_bounds__(SN_THREADS) thin_smalln_kernel(GemmParams p, int kpad) {
  constexpr int R = 32 / NP;
  extern __shared__ __align__(16) float Wt[];   // [NP][kpad]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int idx = tid; idx < NP * kpad; idx += SN_THREADS) {
    int n, k;
    if (NN) { k = idx / NP; n = idx % NP; } else { n = idx / kpad; k = idx % kpad; }
    float v = 0.f;
    if (n < p.N && k < p.K) v = NN ? __ldg(p.B + (long long)k * p.ldb + n) : __ldg(p.B + (long long)n * p.ldb + k);
    Wt[n * kpad + k] = v;
  }
  __syncthreads();
  const int kchunks = kpad >> 7;
  const int groups = (p.M + R - 1) / R;
  const bool needs_z = p.epilogue == EPI_MUL_DTANH || p.epilogue == EPI_ADD_Z;
  for (int g = blockIdx.x * (SN_THREADS / 32) + warp; g < groups; g += gridDim.x * (SN_THREADS / 32)) {
    const int row0 = g * R;
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    for (int j = 0; j < kchunks; ++j) {
      const int k = j * 128 + lane * 4;
      float4 a[R];
#pragma unroll
      for (int r = 0; r < R; ++r) {
        a[r] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (k < p.K && row0 + r < p.M)   // K % 4 == 0 is a dispatch precondition
          a[r] = __ldg(reinterpret_cast<const float4*>(p.A + (long long)(row0 + r) * p.lda + k));
      }
#pragma unroll
      for (int n = 0; n < NP; ++n) {
        const float4 w = *reinterpret_cast<const float4*>(&Wt[n * kpad + k]);
#pragma unroll
        for (int r = 0; r < R; ++r) acc[r * NP + n] = fmaf(a[r].w, w.w, fmaf(a[r].z, w.z, fmaf(a[r].y, w.y, fmaf(a[r].x, w.x, acc[r * NP + n]))));
      }
    }
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
      const bool upper = (lane & off) != 0;
#pragma unroll
      for (int i = 0; i < off; ++i) {
        const float send = upper ? acc[i] : acc[i + off];
        const float keep = upper ? acc[i + off] : acc[i];
        acc[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
      }
    }
    const int row = row0 + lane / NP, n = lane % NP;
    if (row < p.M && n < p.N) {
      const float b = p.bias ? __ldg(p.bias + n) : 0.f;
      const float z = needs_z ? p.Z[(long long)row * p.ldz + n] : 0.f;
      p.C[(long long)row * p.ldc + n] = apply_epilogue(acc[0] + b, p.epilogue, z);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Small-N products whose K is 128 / 256 / 512 (the heads at H = 128..512: N = 1..32 outputs per row).  The kernel
// above keeps 32 accumulators per lane and re-reads the whole [NP][K] weight tile from shared memory for every ROW
// (64 KB of shared-memory traffic per row at K = 512: it runs at the shared-memory roof).  This kernel also keeps the
// [N][K] tile in shared memory, but a warp owns FOUR rows and all 32 lanes share one k-slice layout: lane j holds the
// 16-byte pieces j, j + 32, ... of each of the four rows in registers.  One weight load then feeds four rows, so the
// tile crosses the shared-memory pipe (one quarter warp per clock for 128-bit loads) once per four rows instead of once
// per row.  The 4 x 32 partial sums are reduced with a transposing butterfly: 2 + 1 exchanges halve the rows per lane,
// 3 more add the 8 lanes of a row (6 shuffles per column).
// ------------------------------------------------------------------------------------------------
template <bool NN, int KI>   // KI = K / 32; K / 128 pieces per lane and row
__global__ void __launch_bounds__(256, 2) thin_rowdot4_kernel(GemmParams p) {
  extern __shared__ __align__(16) float Wt[];   // [N][K]
  constexpr int KQ = KI / 4;
  static_assert(KI % 4 == 0, "K must be a multiple of 128");
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int K = KI * 32;
  for (int idx = tid; idx < p.N * K; idx += 256) {
    int n, k;
    if (NN) { k = idx / p.N; n = idx % p.N; } else { n = idx / K; k = idx % K; }
    Wt[n * K + k] = NN ? __ldg(p.B + (long long)k * p.ldb + n) : __ldg(p.B + (long long)n * p.ldb + k);
  }
  __syncthreads();
  const bool needs_z = p.epilogue == EPI_MUL_DTANH || p.epilogue == EPI_ADD_Z;
  const bool hi = (lane & 16) != 0, b8 = (lane & 8) != 0;
  const int my_r = (hi ? 2 : 0) + (b8 ? 1 : 0);   // the row of the group whose sums end up in this lane
  const int groups = (p.M + 3) >> 2;
  for (int g = blockIdx.x * 8 + warp; g < groups; g += gridDim.x * 8) {
    float4 a[4][KQ];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int row = g * 4 + r;
      const bool on = row < p.M;
      const float4* arow = reinterpret_cast<const float4*>(p.A + (long long)(on ? row : 0) * p.lda);
#pragma unroll
      for (int i = 0; i < KQ; ++i) a[r][i] = on ? __ldg(arow + i * 32 + lane) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    const int row = g * 4 + my_r;
    const bool on = row < p.M;
    for (int n = 0; n < p.N; n += 2) {   // two output columns per pass
      const int n1 = n + 1 < p.N ? n + 1 : n;
      const float4* w0 = reinterpret_cast<const float4*>(Wt + n * K);
      const float4* w1 = reinterpret_cast<const float4*>(Wt + n1 * K);
      float s0[4] = {0.f, 0.f, 0.f, 0.f}, s1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int i = 0; i < KQ; ++i) {
        const float4 u = w0[i * 32 + lane], v = w1[i * 32 + lane];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          s0[r] = fmaf(a[r][i].w, u.w, fmaf(a[r][i].z, u.z, fmaf(a[r][i].y, u.y, fmaf(a[r][i].x, u.x, s0[r]))));
          s1[r] = fmaf(a[r][i].w, v.w, fmaf(a[r][i].z, v.z, fmaf(a[r][i].y, v.y, fmaf(a[r][i].x, v.x, s1[r]))));
        }
      }
      // lanes with bit 4 keep rows 2, 3 and hand rows 0, 1 to their partner (and vice versa); then bit 3 picks one row
      float k0 = hi ? s0[2] : s0[0], k1 = hi ? s0[3] : s0[1];
      float l0 = hi ? s1[2] : s1[0], l1 = hi ? s1[3] : s1[1];
      k0 += __shfl_xor_sync(0xffffffffu, hi ? s0[0] : s0[2], 16);
      k1 += __shfl_xor_sync(0xffffffffu, hi ? s0[1] : s0[3], 16);
      l0 += __shfl_xor_sync(0xffffffffu, hi ? s1[0] : s1[2], 16);
      l1 += __shfl_xor_sync(0xffffffffu, hi ? s1[1] : s1[3], 16);
      float acc0 = (b8 ? k1 : k0) + __shfl_xor_sync(0xffffffffu, b8 ? k0 : k1, 8);
      float acc1 = (b8 ? l1 : l0) + __shfl_xor_sync(0xffffffffu, b8 ? l0 : l1, 8);
#pragma unroll
      for (int d = 4; d >= 1; d >>= 1) {
        acc0 += __shfl_xor_sync(0xffffffffu, acc0, d);
        acc1 += __shfl_xor_sync(0xffffffffu, acc1, d);
      }
      // the 8 lanes that hold a row's sums share the stores: lane (n % 8) of them writes column n
      const bool first = (n & 7) == (lane & 7), second = n1 != n && (n1 & 7) == (lane & 7);
      if (on && (first || second)) {
        const int nn = first ? n : n1;
        const float acc = first ? acc0 : acc1;
        const float b = p.bias ? __ldg(p.bias + nn) : 0.f;
        const float z = needs_z ? p.Z[(long long)row * p.ldz + nn] : 0.f;
        p.C[(long long)row * p.ldc + nn] = apply_epilogue(acc + b, p.epilogue, z);
      }
    }
  }
}

template <bool NN, int KI>
int launch_thin_rowdot(const GemmParams& p, cudaStream_t stream) {
  const size_t smem = (size_t)p.N * KI * 32 * sizeof(float);
  static PerDeviceOnce once;
  if (smem > 48 * 1024 && once.need())
    R2D2_CUDA_TRY(cudaFuncSetAttribute(thin_rowdot4_kernel<NN, KI>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
  const int groups = ceil_div(p.M, 4);
  int grid = ceil_div(groups, 8);
  if (grid > num_sms() * 4) grid = num_sms() * 4;
  thin_rowdot4_kernel<NN, KI><<<grid, 256, smem, stream>>>(p);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

// ------------------------------------------------------------------------------------------------
// TN with one small output dimension: X[K rows][P] is the wide operand (thread = one of its columns), Y[K rows][Q<=32]
// the narrow one (staged per 32-row chunk in shared memory, read as broadcast float4).  X rows are fetched sixteen at a
// time (the kernel is latency bound otherwise).  Block column x writes its partial product as slice x of a dense
// C-shaped buffer (the block result goes through shared memory so that the stores walk C in address order whichever
// side is the narrow one); the launcher adds the slices into C in order (split-K contract of gemm_f32: C += A^T B).
// The optional column sums leave the same way: slice x of [P] (X) and of [Q] (Y, blocks with y == 0 only).
// ------------------------------------------------------------------------------------------------
constexpr int TN_THREADS = 256, TN_CHUNK = 32, TN_BATCH = 16;

template <int QP>
__global__ void __launch_bounds__(TN_THREADS) thin_tn_kernel(const float* __restrict__ X, long long ldx, int P,
                                                             const float* __restrict__ Y, long long ldy, int Q, int K,
                                                             float* __restrict__ C_part, int small_is_m,
                                                             float* __restrict__ colsum_x, float* __restrict__ colsum_y) {
  __shared__ __align__(16) float Ys[TN_CHUNK][QP];
  __shared__ float Out[TN_THREADS][QP + 1];
  const int tid = threadIdx.x;
  const int p0 = blockIdx.y * TN_THREADS;
  const int pc = p0 + tid;
  const bool pon = pc < P;
  float acc[QP];
#pragma unroll
  for (int q = 0; q < QP; ++q) acc[q] = 0.f;
  float xsum = 0.f, ysum = 0.f;   // optional column sums of the two operands (bias gradients), each element counted once
  const bool do_ysum = colsum_y != nullptr && blockIdx.y == 0 && tid < Q;
  const int chunks = (K + TN_CHUNK - 1) / TN_CHUNK;
  for (int ch = blockIdx.x; ch < chunks; ch += gridDim.x) {
    const int r0 = ch * TN_CHUNK;
    const int nr = min(TN_CHUNK, K - r0);
    __syncthreads();
    for (int idx = tid; idx < TN_CHUNK * QP; idx += TN_THREADS) {
      const int r = idx / QP, q = idx % QP;
      Ys[r][q] = (r < nr && q < Q) ? __ldg(Y + (long long)(r0 + r) * ldy + q) : 0.f;
    }
    __syncthreads();
    if (do_ysum) {
#pragma unroll 8
      for (int r = 0; r < TN_CHUNK; ++r) ysum += Ys[r][tid];   // rows >= nr hold zeros
    }
    const float* xp = X + (long long)r0 * ldx + pc;
    for (int rb = 0; rb < nr; rb += TN_BATCH) {
      float x[TN_BATCH];
#pragma unroll
      for (int i = 0; i < TN_BATCH; ++i) x[i] = (pon && rb + i < nr) ? __ldg(xp + (long long)(rb + i) * ldx) : 0.f;
#pragma unroll
      for (int i = 0; i < TN_BATCH; ++i) {
        xsum += x[i];
#pragma unroll
        for (int q4 = 0; q4 < QP / 4; ++q4) {
          const float4 y = *reinterpret_cast<const float4*>(&Ys[rb + i][q4 * 4]);   // rows >= nr hold zeros
          acc[q4 * 4 + 0] = fmaf(x[i], y.x, acc[q4 * 4 + 0]); acc[q4 * 4 + 1] = fmaf(x[i], y.y, acc[q4 * 4 + 1]);
          acc[q4 * 4 + 2] = fmaf(x[i], y.z, acc[q4 * 4 + 2]); acc[q4 * 4 + 3] = fmaf(x[i], y.w, acc[q4 * 4 + 3]);
        }
      }
    }
  }
  if (colsum_x && pon) colsum_x[(size_t)blockIdx.x * P + pc] = xsum;
  if (do_ysum) colsum_y[(size_t)blockIdx.x * Q + tid] = ysum;
  float* const C = C_part + (size_t)blockIdx.x * P * Q;   // dense slice: [Q][P] or [P][Q]
#pragma unroll
  for (int q = 0; q < QP; ++q) Out[tid][q] = acc[q];
  __syncthreads();
  const int pn = min(TN_THREADS, P - p0);
  if (small_is_m) {   // C[q][p]: p fastest
    for (int idx = tid; idx < Q * pn; idx += TN_THREADS) {
      const int q = idx / pn, pp = idx % pn;
      C[(long long)q * P + p0 + pp] = Out[pp][q];
    }
  } else {            // C[p][q]: q fastest
    for (int idx = tid; idx < pn * Q; idx += TN_THREADS) {
      const int pp = idx / Q, q = idx % Q;
      C[(long long)(p0 + pp) * Q + q] = Out[pp][q];
    }
  }
}

bool aligned16(const float* ptr, long long ld) {
  return ptr != nullptr && ((reinterpret_cast<uintptr_t>(ptr) & 15) == 0) && (ld % 4 == 0);
}

template <int QP>
int launch_thin_tn(const float* X, long long ldx, int P, const float* Y, long long ldy, int Q, int K, float* C,
                   long long ldc, int small_is_m, float* colsum_x, float* colsum_y, cudaStream_t stream) {
  const int chunks = ceil_div(K, TN_CHUNK), py = ceil_div(P, TN_THREADS);
  int gx = 6 * num_sms() / py;                         // ~6 resident blocks per SM
  if (gx < 1) gx = 1;
  if (gx > chunks) gx = chunks;
  gx = ceil_div(chunks, ceil_div(chunks, gx));         // equal number of chunks per block
  const size_t c_floats = (size_t)gx * P * Q, x_floats = colsum_x ? (size_t)gx * P : 0, y_floats = colsum_y ? (size_t)gx * Q : 0;
  float* part = nullptr;
  R2D2_TRY(partials_scratch(c_floats + x_floats + y_floats, stream, &part));
  float* part_x = colsum_x ? part + c_floats : nullptr;
  float* part_y = colsum_y ? part + c_floats + x_floats : nullptr;
  thin_tn_kernel<QP><<<dim3(gx, py), TN_THREADS, 0, stream>>>(X, ldx, P, Y, ldy, Q, K, part, small_is_m, part_x, part_y);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  if (small_is_m) R2D2_TRY(add_partials(part, gx, Q, P, C, ldc, nullptr, stream));
  else R2D2_TRY(add_partials(part, gx, P, Q, C, ldc, nullptr, stream));
  if (colsum_x) R2D2_TRY(add_partials(part_x, gx, 1, P, colsum_x, P, nullptr, stream));
  if (colsum_y) R2D2_TRY(add_partials(part_y, gx, 1, Q, colsum_y, Q, nullptr, stream));
  return R2D2_OK;
}

int smalln_np(int N) { return N <= 8 ? 8 : N <= 16 ? 16 : 32; }
size_t smalln_smem_bytes(int N, int K) { return (size_t)smalln_np(N) * (ceil_div(K, 128) * 128) * sizeof(float); }

template <bool NN, int NP>
int launch_thin_smalln(const GemmParams& p, cudaStream_t stream) {
  const int kpad = ceil_div(p.K, 128) * 128;
  const size_t smem = smalln_smem_bytes(p.N, p.K);
  if (smem > 48 * 1024)   // rare (N = 32 with K > 384): not worth caching per device
    R2D2_CUDA_TRY(cudaFuncSetAttribute(thin_smalln_kernel<NN, NP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int groups = ceil_div(p.M, 32 / NP);
  int grid = ceil_div(groups, SN_THREADS / 32);
  if (grid > num_sms() * 6) grid = num_sms() * 6;
  thin_smalln_kernel<NN, NP><<<grid, SN_THREADS, smem, stream>>>(p, kpad);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

}  // namespace

// returns R2D2_OK and sets *handled when one of the thin kernels took the problem
int gemm_thin_try(const GemmParams& p, GemmLayout layout, cudaStream_t stream, bool* handled) {
  *handled = false;
  if (layout == GEMM_TN) {
    if (p.split_k <= 1 || p.K2 != 0) return R2D2_OK;          // accumulate-into-zeroed-C contract only
    const bool m_small = p.M <= 32, n_small = p.N <= 32;
    if (!m_small && !n_small) return R2D2_OK;
    // C[m][n] = sum_r A[r][m] B[r][n]
    const bool small_is_m = m_small && (!n_small || p.M <= p.N);
    const float* X = small_is_m ? p.B : p.A;  const long long ldx = small_is_m ? p.ldb : p.lda;
    const float* Y = small_is_m ? p.A : p.B;  const long long ldy = small_is_m ? p.lda : p.ldb;
    const int P = small_is_m ? p.N : p.M, Q = small_is_m ? p.M : p.N;
    float* csx = small_is_m ? p.colsum_b : p.colsum_a;
    float* csy = small_is_m ? p.colsum_a : p.colsum_b;
    *handled = true;
    if (Q <= 8)  return launch_thin_tn<8>(X, ldx, P, Y, ldy, Q, p.K, p.C, p.ldc, small_is_m ? 1 : 0, csx, csy, stream);
    if (Q <= 16) return launch_thin_tn<16>(X, ldx, P, Y, ldy, Q, p.K, p.C, p.ldc, small_is_m ? 1 : 0, csx, csy, stream);
    if (Q <= 24) return launch_thin_tn<24>(X, ldx, P, Y, ldy, Q, p.K, p.C, p.ldc, small_is_m ? 1 : 0, csx, csy, stream);
    return launch_thin_tn<32>(X, ldx, P, Y, ldy, Q, p.K, p.C, p.ldc, small_is_m ? 1 : 0, csx, csy, stream);
  }
  if (p.split_k != 1) return R2D2_OK;
  const bool nn = layout == GEMM_NN;
  if (p.N <= 32 && p.K2 == 0 && (p.K == 128 || p.K == 256 || p.K == 512) && aligned16(p.A, p.lda) &&
      (size_t)p.N * p.K * sizeof(float) <= 64 * 1024) {
    *handled = true;
    if (p.K == 128) return nn ? launch_thin_rowdot<true, 4>(p, stream) : launch_thin_rowdot<false, 4>(p, stream);
    if (p.K == 256) return nn ? launch_thin_rowdot<true, 8>(p, stream) : launch_thin_rowdot<false, 8>(p, stream);
    return nn ? launch_thin_rowdot<true, 16>(p, stream) : launch_thin_rowdot<false, 16>(p, stream);
  }
  // the [NP][kpad] weight tile must fit the opt-in shared memory (N > 16 with K > 1792 on an H100 does not): those
  // products fall through to the mma.sync kernel (N < 32) or wgmma (N = 32)
  if (p.N <= 32 && p.K2 == 0 && p.K >= 64 && p.K <= 2048 && (p.K % 4 == 0) && aligned16(p.A, p.lda) &&
      smalln_smem_bytes(p.N, p.K) <= (size_t)max_smem_optin()) {
    *handled = true;
    if (p.N <= 8)  return nn ? launch_thin_smalln<true, 8>(p, stream) : launch_thin_smalln<false, 8>(p, stream);
    if (p.N <= 16) return nn ? launch_thin_smalln<true, 16>(p, stream) : launch_thin_smalln<false, 16>(p, stream);
    return nn ? launch_thin_smalln<true, 32>(p, stream) : launch_thin_smalln<false, 32>(p, stream);
  }
  if (p.K + p.K2 <= SK_KMAX && (p.K2 == 0 || !nn)) {
    R2D2_REQUIRE(!(p.C_img_k || p.C_img_mn) || (p.N % 32 == 0), "operand image needs N % 32 == 0");
    *handled = true;
    const int row_tiles = ceil_div(p.M, SK_ROWS), ny = ceil_div(p.N, SK_COLS);
    int gx = 3 * num_sms() / ny;                       // 3 resident blocks per SM (registers)
    if (gx < 1) gx = 1;
    if (gx > row_tiles) gx = row_tiles;                // tiles go round-robin over the resident blocks: SM loads differ by <= 1 tile
    const int vec_c = aligned16(p.C, p.ldc) ? 1 : 0, vec_z = aligned16(p.Z, p.ldz) ? 1 : 0;
    if (nn) thin_smallk_kernel<true><<<dim3(gx, ny), SK_THREADS, 0, stream>>>(p, vec_c, vec_z);
    else    thin_smallk_kernel<false><<<dim3(gx, ny), SK_THREADS, 0, stream>>>(p, vec_c, vec_z);
    count_launch();
    R2D2_CUDA_TRY(cudaGetLastError());
    return R2D2_OK;
  }
  return R2D2_OK;
}

}  // namespace r2d2

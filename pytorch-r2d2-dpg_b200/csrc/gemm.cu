// gemm_f32: C = epi(op(A) * op(B) + bias), fp32 in HBM, bf16 hi/lo split in shared memory,
// tensor-core MMAs (3 passes: hi*hi + lo*hi + hi*lo) with fp32 accumulation.
// CTA tile 128x64x32, 8 warps (4 along M x 2 along N), register-staged double buffering.
#include "gemm.cuh"
#include "elementwise.cuh"

#include <stdlib.h>

namespace r2d2 {
namespace {

constexpr int BM = 128, BN = 64, BK = 32, GEMM_THREADS = 256;

template <int LAYOUT>
struct TileGeom {
  static constexpr bool A_KMAJOR = (LAYOUT != GEMM_TN);  // smem A tile [BM][BK] (k contiguous) else [BK][BM]
  static constexpr int A_ROWS = A_KMAJOR ? BM : BK;
  static constexpr int A_COLS = A_KMAJOR ? BK : BM;
  static constexpr int A_LD = A_COLS + 8;                // +16 B pad: conflict-free ldmatrix rows
  static constexpr bool B_KMAJOR = (LAYOUT == GEMM_NT);  // smem B tile [BN][BK] else [BK][BN]
  static constexpr int B_ROWS = B_KMAJOR ? BN : BK;
  static constexpr int B_COLS = B_KMAJOR ? BK : BN;
  static constexpr int B_LD = B_COLS + 8;
  static constexpr int A_PLANE = A_ROWS * A_LD;          // elements (bf16) per hi or lo plane
  static constexpr int B_PLANE = B_ROWS * B_LD;
  static constexpr int STAGE = 2 * A_PLANE + 2 * B_PLANE;
  static constexpr int SMEM_BYTES = 2 * STAGE * (int)sizeof(__nv_bfloat16);
  static constexpr int A_F4_PER_ROW = A_COLS / 4;
  static constexpr int B_F4_PER_ROW = B_COLS / 4;
  static constexpr int A_F4 = A_ROWS * A_COLS / 4 / GEMM_THREADS;  // 4
  static constexpr int B_F4 = B_ROWS * B_COLS / 4 / GEMM_THREADS;  // 2
};

__device__ __forceinline__ float4 guarded_load4(const float* __restrict__ base, long long ld, int row, int col,
                                                int row_lim, int col_lim, bool vec) {
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (row < row_lim && col < col_lim) {
    const float* p = base + (long long)row * ld + col;
    if (vec && col + 3 < col_lim) {
      v = __ldg(reinterpret_cast<const float4*>(p));
    } else {
      v.x = __ldg(p);
      if (col + 1 < col_lim) v.y = __ldg(p + 1);
      if (col + 2 < col_lim) v.z = __ldg(p + 2);
      if (col + 3 < col_lim) v.w = __ldg(p + 3);
    }
  }
  return v;
}

__device__ __forceinline__ void store_split4(__nv_bfloat16* hi_plane, __nv_bfloat16* lo_plane, int off, float4 v) {
  uint32_t h0, l0, h1, l1;
  split_pack2(v.x, v.y, h0, l0);
  split_pack2(v.z, v.w, h1, l1);
  *reinterpret_cast<uint2*>(hi_plane + off) = make_uint2(h0, h1);
  *reinterpret_cast<uint2*>(lo_plane + off) = make_uint2(l0, l1);
}

template <int LAYOUT>
__global__ void __launch_bounds__(GEMM_THREADS)
gemm_bf16x3_kernel(GemmParams p, int vecA, int vecB, int vecA2, int vecB2, long long c_split_stride) {
  using G = TileGeom<LAYOUT>;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __nv_bfloat16* smem = reinterpret_cast<__nv_bfloat16*>(smem_raw);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp & 3, wn = warp >> 2;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;

  const int nk1 = (p.K + BK - 1) / BK;
  const int nk2 = (p.K2 + BK - 1) / BK;
  const int nk_total = nk1 + nk2;
  const int per_split = (nk_total + p.split_k - 1) / p.split_k;
  const int t_begin = blockIdx.z * per_split;
  const int t_end = min(nk_total, t_begin + per_split);
  if (t_begin >= t_end) return;

  float acc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;

  float4 ra[G::A_F4], rb[G::B_F4];

  auto load_tile = [&](int t) {
    const float* Ap; const float* Bp; long long lda, ldb; int k0, klim; bool va, vb;
    if (t < nk1) { Ap = p.A; Bp = p.B; lda = p.lda; ldb = p.ldb; k0 = t * BK; klim = p.K; va = vecA; vb = vecB; }
    else { Ap = p.A2; Bp = p.B2; lda = p.lda2; ldb = p.ldb2; k0 = (t - nk1) * BK; klim = p.K2; va = vecA2; vb = vecB2; }
#pragma unroll
    for (int i = 0; i < G::A_F4; ++i) {
      int q = tid + i * GEMM_THREADS;
      int r = q / G::A_F4_PER_ROW, c = (q % G::A_F4_PER_ROW) * 4;
      if (G::A_KMAJOR) ra[i] = guarded_load4(Ap, lda, m0 + r, k0 + c, p.M, klim, va);
      else             ra[i] = guarded_load4(Ap, lda, k0 + r, m0 + c, klim, p.M, va);
    }
#pragma unroll
    for (int i = 0; i < G::B_F4; ++i) {
      int q = tid + i * GEMM_THREADS;
      int r = q / G::B_F4_PER_ROW, c = (q % G::B_F4_PER_ROW) * 4;
      if (G::B_KMAJOR) rb[i] = guarded_load4(Bp, ldb, n0 + r, k0 + c, p.N, klim, vb);
      else             rb[i] = guarded_load4(Bp, ldb, k0 + r, n0 + c, klim, p.N, vb);
    }
  };

  auto store_tile = [&](int buf) {
    __nv_bfloat16* a_hi = smem + buf * G::STAGE;
    __nv_bfloat16* a_lo = a_hi + G::A_PLANE;
    __nv_bfloat16* b_hi = a_lo + G::A_PLANE;
    __nv_bfloat16* b_lo = b_hi + G::B_PLANE;
#pragma unroll
    for (int i = 0; i < G::A_F4; ++i) {
      int q = tid + i * GEMM_THREADS;
      int r = q / G::A_F4_PER_ROW, c = (q % G::A_F4_PER_ROW) * 4;
      store_split4(a_hi, a_lo, r * G::A_LD + c, ra[i]);
    }
#pragma unroll
    for (int i = 0; i < G::B_F4; ++i) {
      int q = tid + i * GEMM_THREADS;
      int r = q / G::B_F4_PER_ROW, c = (q % G::B_F4_PER_ROW) * 4;
      store_split4(b_hi, b_lo, r * G::B_LD + c, rb[i]);
    }
  };

  auto compute_tile = [&](int buf) {
    const __nv_bfloat16* a_hi = smem + buf * G::STAGE;
    const __nv_bfloat16* a_lo = a_hi + G::A_PLANE;
    const __nv_bfloat16* b_hi = a_lo + G::A_PLANE;
    const __nv_bfloat16* b_lo = b_hi + G::B_PLANE;
    const int j = lane >> 3, r = lane & 7;
#pragma unroll
    for (int kk = 0; kk < BK; kk += 16) {
      uint32_t fa_hi[2][4], fa_lo[2][4], fb_hi[4][2], fb_lo[4][2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        if (G::A_KMAJOR) {
          int off = (wm * 32 + i * 16 + (j & 1) * 8 + r) * G::A_LD + kk + (j >> 1) * 8;
          ldmatrix_x4(fa_hi[i], a_hi + off);
          ldmatrix_x4(fa_lo[i], a_lo + off);
        } else {
          int off = (kk + (j >> 1) * 8 + r) * G::A_LD + wm * 32 + i * 16 + (j & 1) * 8;
          ldmatrix_x4_trans(fa_hi[i], a_hi + off);
          ldmatrix_x4_trans(fa_lo[i], a_lo + off);
        }
      }
#pragma unroll
      for (int pj = 0; pj < 2; ++pj) {
        uint32_t th[4], tl[4];
        if (G::B_KMAJOR) {
          int off = (wn * 32 + pj * 16 + (j >> 1) * 8 + r) * G::B_LD + kk + (j & 1) * 8;
          ldmatrix_x4(th, b_hi + off);
          ldmatrix_x4(tl, b_lo + off);
        } else {
          int off = (kk + (j & 1) * 8 + r) * G::B_LD + wn * 32 + pj * 16 + (j >> 1) * 8;
          ldmatrix_x4_trans(th, b_hi + off);
          ldmatrix_x4_trans(tl, b_lo + off);
        }
        fb_hi[2 * pj][0] = th[0]; fb_hi[2 * pj][1] = th[1]; fb_hi[2 * pj + 1][0] = th[2]; fb_hi[2 * pj + 1][1] = th[3];
        fb_lo[2 * pj][0] = tl[0]; fb_lo[2 * pj][1] = tl[1]; fb_lo[2 * pj + 1][0] = tl[2]; fb_lo[2 * pj + 1][1] = tl[3];
      }
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int jn = 0; jn < 4; ++jn) {
          mma_bf16_16816(acc[i][jn], fa_lo[i], fb_hi[jn]);
          mma_bf16_16816(acc[i][jn], fa_hi[i], fb_lo[jn]);
          mma_bf16_16816(acc[i][jn], fa_hi[i], fb_hi[jn]);
        }
    }
  };

  load_tile(t_begin);
  store_tile(0);
  __syncthreads();
  for (int t = t_begin; t < t_end; ++t) {
    const int buf = (t - t_begin) & 1;
    if (t + 1 < t_end) load_tile(t + 1);
    compute_tile(buf);
    if (t + 1 < t_end) store_tile(buf ^ 1);
    __syncthreads();
  }

  // ---- epilogue ----
  const int g = lane >> 2, c = lane & 3;
  // split-K: slice blockIdx.z of the partial products (c_split_stride floats apart), summed in order by the caller
  float* const C = p.C + (long long)blockIdx.z * c_split_stride;
  const bool vec_c = ((reinterpret_cast<uintptr_t>(C) & 7) == 0) && (p.ldc % 2 == 0);
#pragma unroll
  for (int i = 0; i < 2; ++i) {
#pragma unroll
    for (int jn = 0; jn < 4; ++jn) {
      const int col = n0 + wn * 32 + jn * 8 + 2 * c;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = m0 + wm * 32 + i * 16 + g + h * 8;
        if (row >= p.M || col >= p.N) continue;
        float v0 = acc[i][jn][2 * h], v1 = acc[i][jn][2 * h + 1];
        const bool has1 = (col + 1 < p.N);
        if (p.bias) { v0 += __ldg(p.bias + col); if (has1) v1 += __ldg(p.bias + col + 1); }
        if (p.epilogue == EPI_TANH) { v0 = tanhf(v0); v1 = tanhf(v1); }
        else if (p.epilogue == EPI_MUL_DTANH) {
          const float* z = p.Z + (long long)row * p.ldz + col;
          float z0 = z[0]; v0 *= (1.f - z0 * z0);
          if (has1) { float z1 = z[1]; v1 *= (1.f - z1 * z1); }
        } else if (p.epilogue == EPI_ADD_Z) {
          const float* z = p.Z + (long long)row * p.ldz + col;
          v0 += z[0];
          if (has1) v1 += z[1];
        }
        float* cp = C + (long long)row * p.ldc + col;
        if (vec_c && has1) {
          *reinterpret_cast<float2*>(cp) = make_float2(v0, v1);
        } else {
          cp[0] = v0;
          if (has1) cp[1] = v1;
        }
      }
    }
  }
}

template <int LAYOUT>
int launch_gemm(const GemmParams& p, cudaStream_t stream) {
  using G = TileGeom<LAYOUT>;
  static PerDeviceOnce once;
  if (once.need()) {
    R2D2_CUDA_TRY(cudaFuncSetAttribute(gemm_bf16x3_kernel<LAYOUT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       G::SMEM_BYTES));
  }
  auto aligned = [](const float* ptr, long long ld) {
    return ptr != nullptr && ((reinterpret_cast<uintptr_t>(ptr) & 15) == 0) && (ld % 4 == 0);
  };
  GemmParams q = p;
  int slices = 1;
  if (p.split_k > 1) {   // partial products into slices, then added into C in slice order (same bits every run)
    const int nk = ceil_div(p.K, BK) + ceil_div(p.K2, BK), per_split = ceil_div(nk, p.split_k);
    slices = ceil_div(nk, per_split);                    // every slice z < slices owns at least one k tile
    R2D2_TRY(partials_scratch((size_t)slices * p.M * p.N, stream, &q.C));
    q.ldc = p.N;
  }
  dim3 grid(ceil_div(p.N, BN), ceil_div(p.M, BM), slices);
  gemm_bf16x3_kernel<LAYOUT><<<grid, GEMM_THREADS, G::SMEM_BYTES, stream>>>(
      q, aligned(p.A, p.lda), aligned(p.B, p.ldb), aligned(p.A2, p.lda2), aligned(p.B2, p.ldb2), (long long)p.M * p.N);
  count_launch();
  R2D2_CUDA_TRY(cudaGetLastError());
  if (p.split_k > 1) return add_partials(q.C, slices, p.M, p.N, p.C, p.ldc, nullptr, stream);
  return R2D2_OK;
}

}  // namespace

static int g_gemm_impl = -1;
void gemm_set_impl(int impl) { g_gemm_impl = impl ? 1 : 0; }
int gemm_get_impl() {
  if (g_gemm_impl < 0) {
    const char* e = getenv("R2D2_GEMM_IMPL");
    g_gemm_impl = (e && (e[0] == 'm' || e[0] == '0')) ? 0 : 1;
  }
  return g_gemm_impl;
}

static int g_skinny_mma = 1;
void gemm_set_impl_skinny_mma(int on) { g_skinny_mma = on ? 1 : 0; }
int gemm_get_impl_skinny_mma() { return g_skinny_mma; }

bool gemm_supports_bias2(int M, int N, int K) {
  const bool skinny = (K < 64) || (N < 32) || (M < 32);
  return gemm_get_impl() == 1 && !(skinny && gemm_get_impl_skinny_mma());
}

bool gemm_emits_operand_image(int M, int N, int K_total) {
  if (gemm_get_impl() != 1 || N <= 32 || N % 32 != 0) return false;
  if (gemm_get_impl_skinny_mma() && K_total <= 32) return true;                 // small-K streaming kernel (gemm_thin.cu)
  const bool skinny = (K_total < 64) || (M < 32);
  return !(skinny && gemm_get_impl_skinny_mma());                              // wgmma epilogue (gemm_tc.cu)
}

int gemm_suggest_split_k(int M, int N, int K) {
  const bool skinny = (K < 64) || (N < 32) || (M < 32);
  if (gemm_get_impl() == 1 && !(skinny && g_skinny_mma)) return gemm_tc_suggest_split_k(M, N, K);
  long long tiles = (long long)ceil_div(M, BM) * ceil_div(N, BN);
  int k_tiles = ceil_div(K, BK);
  if (tiles >= num_sms() || k_tiles < 16) return 1;
  int want = (int)ceil_div_ll(2 * num_sms(), tiles);
  int max_by_k = k_tiles / 8;  // keep >= 8 k-tiles (256 k) per split
  int s = want < max_by_k ? want : max_by_k;
  if (s < 1) s = 1;
  if (s > 128) s = 128;
  return s;
}

static int gemm_f32_dispatch(const GemmParams& p, GemmLayout layout, cudaStream_t stream, bool* colsums_done);

int gemm_f32(const GemmParams& p, GemmLayout layout, cudaStream_t stream) {
  R2D2_REQUIRE((!p.colsum_a && !p.colsum_b) || layout == GEMM_TN, "column sums ride on TN products only");
  bool colsums_done = false;
  R2D2_TRY(gemm_f32_dispatch(p, layout, stream, &colsums_done));
  if (!colsums_done) {   // the kernel that took the product does not fuse them
    if (p.colsum_a) R2D2_TRY(colsum(p.A, p.lda, p.K, p.M, p.colsum_a, nullptr, stream));
    if (p.colsum_b) R2D2_TRY(colsum(p.B, p.ldb, p.K, p.N, p.colsum_b, nullptr, stream));
  }
  return R2D2_OK;
}

static int gemm_f32_dispatch(const GemmParams& p, GemmLayout layout, cudaStream_t stream, bool* colsums_done) {
  R2D2_REQUIRE((p.A || p.A_img) && (p.B || p.B_img) && p.C, "null operand");
  if (p.A_img || p.B_img) {
    R2D2_REQUIRE(p.K2 == 0, "packed A with a second K segment");
    return gemm_f32_tc(p, layout, stream);
  }
  R2D2_REQUIRE(p.M > 0 && p.N > 0 && p.K > 0, "empty problem");
  R2D2_REQUIRE(p.split_k >= 1, "split_k");
  R2D2_REQUIRE(p.split_k == 1 || (p.epilogue == EPI_NONE && p.bias == nullptr), "split-K supports no epilogue");
  R2D2_REQUIRE(p.K2 == 0 || layout == GEMM_NT, "second K segment only for NT");
  R2D2_REQUIRE(p.K2 == 0 || (p.A2 && p.B2), "segment 2 operands");
  R2D2_REQUIRE((p.epilogue != EPI_MUL_DTANH && p.epilogue != EPI_ADD_Z) || p.Z, "epilogue needs Z");
  R2D2_REQUIRE(ceil_div(p.M, BM) <= 65535, "M too large for grid.y");
  // skinny problems (K < 64: obs/act inputs; N < 32: heads, dW1/dW3 blocks) are launch/latency bound: the single-launch
  // mma.sync kernel beats pack + pack + wgmma there (tools/gemm_bench.py); everything else goes to the wgmma path
  const bool skinny = (p.K + p.K2 < 64) || (p.N < 32) || (p.M < 32);
  if (gemm_get_impl() == 1 && gemm_get_impl_skinny_mma()) {   // default mode: degenerate shapes -> fp32 streaming kernels
    bool handled = false;
    R2D2_TRY(gemm_thin_try(p, layout, stream, &handled));
    if (handled) { *colsums_done = true; return R2D2_OK; }
  }
  R2D2_REQUIRE(!p.bias2 || gemm_supports_bias2(p.M, p.N, p.K + p.K2), "bias2 needs the wgmma path (gemm_supports_bias2)");
  R2D2_REQUIRE((!p.C_img_k && !p.C_img_mn) || (layout == GEMM_NT && gemm_emits_operand_image(p.M, p.N, p.K + p.K2)),
               "C_img_* is produced by the small-K streaming kernel and the wgmma epilogue only (see gemm_emits_operand_image)");
  if (gemm_get_impl() == 1 && !(skinny && gemm_get_impl_skinny_mma())) return gemm_f32_tc(p, layout, stream);
  switch (layout) {
    case GEMM_NT: return launch_gemm<GEMM_NT>(p, stream);
    case GEMM_NN: return launch_gemm<GEMM_NN>(p, stream);
    case GEMM_TN: return launch_gemm<GEMM_TN>(p, stream);
  }
  set_last_error("bad gemm layout");
  return R2D2_ERR_ARG;
}

}  // namespace r2d2

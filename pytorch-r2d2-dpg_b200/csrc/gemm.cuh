// General fp32-in / fp32-out GEMM on tensor cores with bf16 hi/lo operand split (3 MMA passes,
// fp32 accumulate) - the dense contractions of the learner path that are NOT on the serial chain:
//   x*W1^T, z*W_ih^T, heads (models.py:33,37-39,76,80-82) and their dgrad / wgrad twins.
#pragma once
#include "common.cuh"

namespace r2d2 {

enum GemmLayout : int {
  GEMM_NT = 0,  // A[M,K] row-major, B[N,K] row-major : C = A * B^T   (forward linear, weights [out,in])
  GEMM_NN = 1,  // A[M,K] row-major, B[K,N] row-major : C = A * B     (dgrad: dY[M,out] * W[out,in])
  GEMM_TN = 2   // A[K,M] row-major, B[K,N] row-major : C = A^T * B   (wgrad: dY^T * X, K = T*B rows)
};

enum GemmEpilogue : int {
  EPI_NONE = 0,
  EPI_TANH = 1,        // C = tanh(acc + bias)
  EPI_MUL_DTANH = 2,   // C = (acc + bias) * (1 - Z^2)
  EPI_ADD_Z = 3        // C = acc + bias + Z
};

struct GemmParams {
  const float* A = nullptr;  long long lda = 0;
  const float* B = nullptr;  long long ldb = 0;
  // optional second K segment (GEMM_NT only): C += A2[M,K2] * B2[N,K2]^T  (critic input = cat(obs, act))
  const float* A2 = nullptr; long long lda2 = 0;
  const float* B2 = nullptr; long long ldb2 = 0;
  int K2 = 0;
  float* C = nullptr;        long long ldc = 0;
  int M = 0, N = 0, K = 0;
  const float* bias = nullptr;          // [N]
  const float* bias2 = nullptr;         // [N] second bias added to the first (b_ih + b_hh); wgmma path only, see
                                        // gemm_supports_bias2
  const float* Z = nullptr;  long long ldz = 0;   // [M,N] aux for the epilogue
  int epilogue = EPI_NONE;
  int split_k = 1;           // >1: K split over CTAs; the partial products are added into C in split order
  const unsigned char* A_img = nullptr;   // wgmma path: A already in packed tile-major form (gemm_tc.cu image of this
                             // call's layout and tiling, e.g. written by the BPTT scan); A / lda are ignored
  unsigned char* C_img_k = nullptr;      // NT, N % 32 == 0 (gemm_emits_operand_image): also write C as the K-major packed operand image
                             // [ceil(M/128)][N/32][16 KB] for a following product that contracts over N
  unsigned char* C_img_mn = nullptr;     // same, MN-major image [ceil(N/128)][ceil(M/32)][16 KB]: C as the B operand of a TN
                             // product that contracts over C's rows (z1 in dW_ih)
  const unsigned char* B_img = nullptr;   // wgmma path: B already packed (image of this call's layout and tiling)
  float* colsum_a = nullptr;             // TN only: also ADD the column sums of A[K,M] (M values) / B[K,N] (N values) here:
  float* colsum_b = nullptr;             // the bias gradient that goes with a weight gradient reads the same rows
  int reuse_packed_a = 0;    // wgmma path: A (pointer, shape, layout) is the operand the previous gemm_f32 call packed
                             // and its contents have not changed since -> skip the pack pass (dW_hh then dW_ih of a chain)
};

int gemm_f32(const GemmParams& p, GemmLayout layout, cudaStream_t stream);
// true when gemm_f32 will honour GemmParams::C_img_k / C_img_mn for an NT product with these sizes (the small-K streaming
// kernel or the wgmma epilogue is selected)
bool gemm_emits_operand_image(int M, int N, int K_total);
// true when gemm_f32 will take this NT product on the wgmma path, which honours GemmParams::bias2
bool gemm_supports_bias2(int M, int N, int K);
// picks a split-K factor so that a skinny-output wgrad GEMM fills the SMs
int gemm_suggest_split_k(int M, int N, int K);

// implementation: 1 = wgmma kernel (default), 0 = mma.sync kernel; env R2D2_GEMM_IMPL = "tc" | "mma"
void gemm_set_impl(int impl);
int gemm_get_impl();
// with the wgmma implementation selected, skinny problems still take the single-launch mma.sync kernel (default on)
void gemm_set_impl_skinny_mma(int on);
int gemm_get_impl_skinny_mma();
int gemm_f32_tc(const GemmParams& p, GemmLayout layout, cudaStream_t stream);
// fp32 streaming kernels for contractions with one dimension <= 32 (gemm_thin.cu); *handled = false when the shape is
// not one of theirs
int gemm_thin_try(const GemmParams& p, GemmLayout layout, cudaStream_t stream, bool* handled);
int gemm_tc_suggest_split_k(int M, int N, int K);

}  // namespace r2d2

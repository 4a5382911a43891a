#include "net.cuh"

#include "elementwise.cuh"
#include "gemm.cuh"
#include "lstm_scan.cuh"

namespace r2d2 {

static size_t align64(size_t n) { return (n + 63) & ~(size_t)63; }  // 256-byte aligned sub-buffers
static size_t pad_to(size_t n, size_t m) { return (n + m - 1) / m * m; }

size_t ChainWs::floats(const NetShape& s, int T, int B, int repeat) {
  const size_t H = s.hidden, A = s.act, S = (size_t)T * repeat, TB = (size_t)T * B;
  size_t n = 0;
  n += align64(TB * H);                        // z1
  n += align64(TB * 4 * H);                    // gin
  if (repeat > 1) n += align64(S * B * 4 * H); // gates
  n += 2 * align64((S + 1) * B * H);           // hs, cs
  n += align64(TB * H);                        // head_in
  n += align64(TB * H);                        // dh_head
  n += 2 * align64(TB * A);                    // head_out, d_pre
  n += align64(4 * H);                         // bias_sum
  size_t sc = lstm_scan_fwd_scratch_floats(B, s.hidden);
  const size_t sb = lstm_scan_bwd_scratch_floats(B, s.hidden);
  if (sb > sc) sc = sb;
  n += align64(sc + 64);
  n += align64(pad_to(TB, 128) * H);           // z1 operand image (bf16 hi + lo: 4 bytes per element)
  return n;
}

ChainWs ChainWs::carve(float* base, const NetShape& s, int T, int B, int repeat) {
  const size_t H = s.hidden, A = s.act, S = (size_t)T * repeat, TB = (size_t)T * B;
  ChainWs w;
  float* p = base;
  auto take = [&](size_t n) { float* r = p; p += align64(n); return r; };
  w.z1 = take(TB * H);
  w.gin = take(TB * 4 * H);
  w.gates = (repeat > 1) ? take(S * B * 4 * H) : w.gin;
  w.hs = take((S + 1) * B * H);
  w.cs = take((S + 1) * B * H);
  w.head_in = take(TB * H);
  w.dh_head = take(TB * H);
  w.head_out = take(TB * A);
  w.d_pre = take(TB * A);
  w.bias_sum = take(4 * H);
  size_t sc = lstm_scan_fwd_scratch_floats(B, s.hidden);
  const size_t sb = lstm_scan_bwd_scratch_floats(B, s.hidden);
  if (sb > sc) sc = sb;
  w.scratch = take(sc + 64);
  w.img_k = reinterpret_cast<unsigned char*>(take(pad_to(TB, 128) * H));
  return w;
}

int net_forward(const NetShape& s, const NetParams& P, const ChainWs& ws, const float* obs, const float* act,
                const float* h0, const float* c0, int T, int B, int repeat, cudaStream_t stream) {
  R2D2_TRY(net_forward_inputs(s, P, ws, obs, act, T, B, stream));
  return net_forward_scan(s, P, ws, h0, c0, T, B, repeat, stream);
}

// The non-recurrent half of a chain: z1 = tanh(l1(x)) and gin = z1 * W_ih^T + b_ih + b_hh for all rows at once.  It
// depends on the inputs and the weights only, so a caller may run it on another stream long before the scan.
int net_forward_inputs(const NetShape& s, const NetParams& P, const ChainWs& ws, const float* obs, const float* act,
                       int T, int B, cudaStream_t stream) {
  const int H = s.hidden, O = s.obs, A = s.act, I = s.in_features();
  const int M = T * B;
  R2D2_REQUIRE(!s.critic || act != nullptr, "critic needs actions");
  bool z1_img = false;
  {  // z1 = tanh(x * W1^T + b1)   (models.py:33 / :75-76; cat(obs, act) as two K segments)
    GemmParams g;
    g.A = obs; g.lda = O; g.B = P.w1; g.ldb = I; g.K = O;
    if (s.critic) { g.A2 = act; g.lda2 = A; g.B2 = P.w1 + O; g.ldb2 = I; g.K2 = A; }
    g.C = ws.z1; g.ldc = H; g.M = M; g.N = H; g.bias = P.b1; g.epilogue = EPI_TANH;
    // the l1 kernel can write z1 a second time as the packed A operand of the W_ih product
    z1_img = ws.img_k != nullptr && gemm_emits_operand_image(M, H, I);
    if (z1_img) g.C_img_k = ws.img_k;
    R2D2_TRY(gemm_f32(g, GEMM_NT, stream));
  }
  const bool two_bias = gemm_supports_bias2(M, 4 * H, H);   // the wgmma epilogue adds both biases itself
  if (!two_bias) R2D2_TRY(add_vec(P.bih, P.bhh, ws.bias_sum, 4 * H, stream));
  {  // gin = z1 * W_ih^T + (b_ih + b_hh)   (input half of LSTMCell, models.py:37,80) for all rows at once
    GemmParams g;
    g.A = ws.z1; g.lda = H; g.B = P.wih; g.ldb = H; g.K = H;
    g.C = ws.gin; g.ldc = 4 * H; g.M = M; g.N = 4 * H;
    if (two_bias) { g.bias = P.bih; g.bias2 = P.bhh; } else g.bias = ws.bias_sum;
    if (z1_img) g.A_img = ws.img_k;
    R2D2_TRY(gemm_f32(g, GEMM_NT, stream));
  }
  return R2D2_OK;
}

int net_forward_scan(const NetShape& s, const NetParams& P, const ChainWs& ws, const float* h0, const float* c0, int T,
                     int B, int repeat, cudaStream_t stream) {
  const int H = s.hidden;
  ScanFwdParams sp;
  sp.gin = ws.gin; sp.whh = P.whh; sp.h0 = h0; sp.c0 = c0;
  sp.gates = ws.gates; sp.hs = ws.hs; sp.cs = ws.cs;
  sp.head_in = s.critic ? nullptr : ws.head_in;
  sp.T = T; sp.B = B; sp.H = H; sp.repeat = repeat; sp.scratch = ws.scratch;
  sp.no_save = ws.inference_only ? 1 : 0;
  return lstm_scan_forward(sp, stream);
}

static const float* head_input(const NetShape& s, const ChainWs& ws, int first_row, int B) {
  // actor: tanh(h) rows saved by the scan; critic: h itself (models.py:82 reads self.hx, the tanh at :81 is dropped)
  return s.critic ? ws.hs + (size_t)(1 + first_row) * B * s.hidden : ws.head_in + (size_t)first_row * B * s.hidden;
}

int net_head_forward(const NetShape& s, const NetParams& P, const ChainWs& ws, int first_row, int T, int B,
                     int repeat, float* out, long long ldo, cudaStream_t stream) {
  R2D2_REQUIRE(!s.critic || repeat == 1, "critic chains run one cell step per row");
  R2D2_REQUIRE(first_row >= 0 && first_row < T, "head_first_row");
  GemmParams g;
  g.A = head_input(s, ws, first_row, B); g.lda = s.hidden;
  g.B = P.w3; g.ldb = s.hidden; g.K = s.hidden;
  g.C = out; g.ldc = ldo; g.M = (T - first_row) * B; g.N = s.act; g.bias = P.b3;
  g.epilogue = s.critic ? EPI_NONE : EPI_TANH;
  return gemm_f32(g, GEMM_NT, stream);
}

int net_backward(const NetShape& s, const NetParams& P, const NetParams* G, const ChainWs& ws, const float* obs,
                 const float* act, const float* d_pre, int first_row, int T, int B, int repeat, float* d_act,
                 const float* dact_z, cudaStream_t stream) {
  const int H = s.hidden, O = s.obs, A = s.act, I = s.in_features();
  const int S = T * repeat, M = T * B, Mh = (T - first_row) * B;
  R2D2_REQUIRE(!s.critic || repeat == 1, "critic chains run one cell step per row");
  const float* hin = head_input(s, ws, first_row, B);
  if (G) {  // head weight / bias gradients
    GemmParams g;
    g.A = d_pre; g.lda = A; g.B = hin; g.ldb = H; g.K = Mh;
    g.C = G->w3; g.ldc = H; g.M = A; g.N = H; g.split_k = gemm_suggest_split_k(A, H, Mh);
    g.colsum_a = G->b3;   // db3 = column sums of d_pre: same rows, same pass
    R2D2_TRY(gemm_f32(g, GEMM_TN, stream));
  }
  {  // dL/dh from the head: d_pre * W3 (actor: through tanh(h), models.py:38)
    GemmParams g;
    g.A = d_pre; g.lda = A; g.B = P.w3; g.ldb = H; g.K = A;
    g.C = ws.dh_head; g.ldc = H; g.M = Mh; g.N = H;
    if (!s.critic) { g.Z = hin; g.ldz = H; g.epilogue = EPI_MUL_DTANH; }
    R2D2_TRY(gemm_f32(g, GEMM_NN, stream));
  }
  float* dgin = (repeat > 1) ? ws.gin : ws.gates;
  {
    ScanBwdParams bp;
    bp.gates = ws.gates; bp.hs = ws.hs; bp.cs = ws.cs; bp.whh = P.whh;
    bp.dh_head = ws.dh_head; bp.head_first_step = first_row * repeat;
    bp.dgates = ws.gates; bp.dgin = dgin;
    bp.T = T; bp.B = B; bp.H = H; bp.repeat = repeat; bp.scratch = ws.scratch;
    if (G) { bp.dbias = G->bih; bp.dbias2 = G->bhh; }   // db_ih = db_hh = sum of dG, accumulated inside the scan
    R2D2_TRY(lstm_scan_backward(bp, stream));
  }
  if (G) {
    {  // dW_hh = sum_s dG_s^T h_{s-1}
      GemmParams g;
      g.A = ws.gates; g.lda = 4 * H; g.B = ws.hs; g.ldb = H; g.K = S * B;
      g.C = G->whh; g.ldc = H; g.M = 4 * H; g.N = H; g.split_k = gemm_suggest_split_k(4 * H, H, S * B);
      R2D2_TRY(gemm_f32(g, GEMM_TN, stream));
    }
    {  // dW_ih = sum_t dGin_t^T z1_t
      GemmParams g;
      g.A = dgin; g.lda = 4 * H; g.B = ws.z1; g.ldb = H; g.K = M;
      g.C = G->wih; g.ldc = H; g.M = 4 * H; g.N = H; g.split_k = gemm_suggest_split_k(4 * H, H, M);
      g.reuse_packed_a = (repeat == 1);   // same dG operand as the dW_hh product just above
      R2D2_TRY(gemm_f32(g, GEMM_TN, stream));
    }
  }
  {  // d(pre-l1) = (dGin * W_ih) * (1 - z1^2), in place over z1
    GemmParams g;
    g.A = dgin; g.lda = 4 * H; g.B = P.wih; g.ldb = H; g.K = 4 * H;
    g.C = ws.z1; g.ldc = H; g.M = M; g.N = H; g.Z = ws.z1; g.ldz = H; g.epilogue = EPI_MUL_DTANH;
    R2D2_TRY(gemm_f32(g, GEMM_NN, stream));
  }
  if (G) {
    GemmParams g;
    g.A = ws.z1; g.lda = H; g.B = obs; g.ldb = O; g.K = M;
    g.C = G->w1; g.ldc = I; g.M = H; g.N = O; g.split_k = gemm_suggest_split_k(H, O, M);
    g.colsum_a = G->b1;   // db1 = column sums of d(pre-l1)
    R2D2_TRY(gemm_f32(g, GEMM_TN, stream));
    if (s.critic) {
      GemmParams g2 = g;
      g2.colsum_a = nullptr;
      g2.B = act; g2.ldb = A; g2.C = G->w1 + O; g2.N = A; g2.split_k = gemm_suggest_split_k(H, A, M);
      R2D2_TRY(gemm_f32(g2, GEMM_TN, stream));
    }
  }
  if (d_act) {  // gradient wrt the action half of the critic input (DPG path, learner.py:123-127)
    R2D2_REQUIRE(s.critic, "d_act only for the critic");
    GemmParams g;
    g.A = ws.z1; g.lda = H; g.B = P.w1 + O; g.ldb = I; g.K = H;
    g.C = d_act; g.ldc = A; g.M = M; g.N = A;
    if (dact_z) { g.Z = dact_z; g.ldz = A; g.epilogue = EPI_MUL_DTANH; }
    R2D2_TRY(gemm_f32(g, GEMM_NN, stream));
  }
  return R2D2_OK;
}

}  // namespace r2d2

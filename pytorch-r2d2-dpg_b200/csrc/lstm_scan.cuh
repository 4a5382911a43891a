// Serial part of the recurrent nets (models.py:37,80 `self.l2(x,(hx,cx))` unrolled over the whole
// burn-in + learning window, learner.py:92-109,120-123) as ONE persistent launch per chain:
//   gates_s = gin[s/repeat] + h_{s-1} * W_hh^T ; (i,f,g,o) ; c_s = f*c_{s-1} + i*g ; h_s = o*tanh(c_s)
// and its BPTT twin.  The non-recurrent x*W_ih^T + b_ih + b_hh is hoisted into `gin` by gemm_f32.
#pragma once
#include "common.cuh"

namespace r2d2 {

struct ScanFwdParams {
  const float* gin = nullptr;   // [T,B,4H] pre-activation input projection (+ both biases)
  const float* whh = nullptr;   // [4H,H]  (torch LSTMCell weight_hh, gate order i,f,g,o)
  const float* h0 = nullptr;    // [B,H] or null (zero state, models.py:34-36)
  const float* c0 = nullptr;
  float* gates = nullptr;       // [S,B,4H] post-activation gates (may alias gin when repeat == 1)
  float* hs = nullptr;          // [S+1,B,H]; slot 0 = initial state
  float* cs = nullptr;          // [S+1,B,H]
  float* head_in = nullptr;     // optional [T,B,H]: tanh(h) at steps s % repeat == repeat-1 (actor head input)
  int T = 0, B = 0, H = 0, repeat = 1;   // S = T*repeat; repeat=2 reproduces the double actor step (learner.py:122-123)
  float* scratch = nullptr;     // per-step path: [B,4H]
  int no_save = 0;              // 1: chain is never back-propagated (target nets): the cluster kernels store neither gates
                                // nor cs[1..S] (hs and head_in are stored)
};

struct ScanBwdParams {
  const float* gates = nullptr;    // [S,B,4H] saved by the forward scan
  const float* hs = nullptr;       // [S+1,B,H]
  const float* cs = nullptr;       // [S+1,B,H]
  const float* whh = nullptr;      // [4H,H]
  const float* dh_head = nullptr;  // [*,B,H] dLoss/dh from the head; row (s-head_first_step)/repeat is consumed at
                                   // step s when s >= head_first_step and (s-head_first_step) % repeat == repeat-1
  int head_first_step = 0;         // burn-in steps carry no head gradient (learner.py:93 vs :105)
  float* dgates = nullptr;         // [S,B,4H] dLoss/d(pre-activation gates) (may alias gates)
  float* dgin = nullptr;           // [T,B,4H] sum over the `repeat` steps sharing an input row (== dgates if repeat==1)
  int T = 0, B = 0, H = 0, repeat = 1;
  float* scratch = nullptr;        // per-step path: [2,B,H] (dh_rec, dc)
  float* dbias = nullptr;          // optional [4H]: column sums of dgates over all steps and rows are ADDED here
  float* dbias2 = nullptr;         // optional second copy (b_ih and b_hh receive the same gradient)
};

// true when persistent cluster kernels cover this hidden size (H in {32,64,128,256,512})
bool lstm_scan_cluster_supported(int H);
int lstm_scan_forward(const ScanFwdParams& p, cudaStream_t stream);
int lstm_scan_backward(const ScanBwdParams& p, cudaStream_t stream);
// per-step path scratch requirements in floats (reserved for every H: the path can be selected at run time)
size_t lstm_scan_fwd_scratch_floats(int B, int H);
size_t lstm_scan_bwd_scratch_floats(int B, int H);

// 1 = persistent cluster kernels where they cover H (default), 0 = per-step path (one GEMM + one cell kernel per step)
// for every H, the A/B reference.  Initialised from the environment variable R2D2_SCAN_IMPL ("cluster" | "step").
void lstm_scan_set_impl(int impl);
int lstm_scan_get_impl();
// nonzero if a bounded hand-off wait inside a cluster scan kernel expired (the word stays set for the rest of the
// process: the results of that launch and of later ones are not to be trusted); synchronises the stream
int lstm_scan_error_status(int* out, cudaStream_t stream);

}  // namespace r2d2

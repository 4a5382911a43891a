// One recurrent net chain = hoisted dense GEMMs + persistent scan + head, and its BPTT.
// Restates ActorNet/CriticNet.__call__ (models.py:32-40,74-83) unrolled over a window of rows.
#pragma once
#include "common.cuh"

namespace r2d2 {

struct NetShape {
  int obs = 0, act = 0, hidden = 0;
  bool critic = false;
  int in_features() const { return obs + (critic ? act : 0); }
  size_t param_count() const {
    const size_t H = hidden, I = in_features(), A = act;
    return H * I + H + 4 * H * H * 2 + 4 * H * 2 + A * H + A;
  }
};

// views into a flat parameter (or gradient) block, reference state_dict order (models.py:17-19,59-61)
struct NetParams {
  float *w1, *b1, *wih, *whh, *bih, *bhh, *w3, *b3;
  static NetParams from_flat(float* flat, const NetShape& s) {
    const size_t H = s.hidden, I = s.in_features(), A = s.act;
    NetParams p;
    p.w1 = flat;            p.b1 = p.w1 + H * I;
    p.wih = p.b1 + H;       p.whh = p.wih + 4 * H * H;
    p.bih = p.whh + 4 * H * H; p.bhh = p.bih + 4 * H;
    p.w3 = p.bhh + 4 * H;   p.b3 = p.w3 + A * H;
    return p;
  }
};

// activations of one chain (carved from one workspace block)
struct ChainWs {
  float* z1 = nullptr;        // [T,B,H] tanh(l1(x)); overwritten by d(pre-l1) in the backward pass
  float* gin = nullptr;       // [T,B,4H] input projection (aliases gates when repeat == 1); dgin in backward
  float* gates = nullptr;     // [S,B,4H] post-activation gates; dgates in backward
  float* hs = nullptr;        // [S+1,B,H]
  float* cs = nullptr;        // [S+1,B,H]
  float* head_in = nullptr;   // [T,B,H] tanh(h) at the last step of each row (actor only)
  float* dh_head = nullptr;   // [T,B,H]
  float* head_out = nullptr;  // [T,B,A] (kept for the C-ABI entry: actor dtanh)
  float* d_pre = nullptr;     // [T,B,A]
  float* bias_sum = nullptr;  // [4H] b_ih + b_hh
  float* scratch = nullptr;   // generic scan path
  unsigned char* img_k = nullptr;       // z1 as the packed K-major A operand of z1 * W_ih^T (written by the l1 kernel)
  bool inference_only = false;          // set by the owner of a chain that is never back-propagated (target nets)
  static size_t floats(const NetShape& s, int T, int B, int repeat);
  static ChainWs carve(float* base, const NetShape& s, int T, int B, int repeat);
};

// forward over T rows (S = T*repeat steps).  obs [T*B, O], act [T*B, A] (critic).
int net_forward(const NetShape& s, const NetParams& P, const ChainWs& ws, const float* obs, const float* act,
                const float* h0, const float* c0, int T, int B, int repeat, cudaStream_t stream);
// the two halves of net_forward: hoisted input GEMMs (inputs + weights only) and the recurrent scan
int net_forward_inputs(const NetShape& s, const NetParams& P, const ChainWs& ws, const float* obs, const float* act,
                       int T, int B, cudaStream_t stream);
int net_forward_scan(const NetShape& s, const NetParams& P, const ChainWs& ws, const float* h0, const float* c0, int T,
                     int B, int repeat, cudaStream_t stream);
// head on rows [first_row, T): out [(T-first_row)*B, A] with leading dimension ldo
int net_head_forward(const NetShape& s, const NetParams& P, const ChainWs& ws, int first_row, int T, int B,
                     int repeat, float* out, long long ldo, cudaStream_t stream);
// BPTT.  d_pre [(T-first_row)*B, A] = dLoss/d(head pre-activation).  G: gradient views (pre-zeroed, accumulated)
// or nullptr for data-gradient only.  d_act [T*B, A] optional (critic): dLoss/d(action input), multiplied by
// (1 - dact_z^2) when dact_z is given (fuses the actor's output tanh, models.py:39).
int net_backward(const NetShape& s, const NetParams& P, const NetParams* G, const ChainWs& ws, const float* obs,
                 const float* act, const float* d_pre, int first_row, int T, int B, int repeat, float* d_act,
                 const float* dact_z, cudaStream_t stream);

}  // namespace r2d2

// Persistent LSTM scan kernels (forward + BPTT) for sm_90a.
//
// Decomposition (H in {32,64,128,256,512}):  a thread-block cluster of C = H/32 CTAs owns NB batch
// rows for the whole chain.  CTA `rank` owns hidden units [32*rank, 32*rank+32): its 128 gate rows of
// W_hh stay resident as bf16 hi/lo MMA fragments for the whole launch (loaded once) - in REGISTERS up to H = 256;
// at H = 512 (cluster of 16, non-portable size) the slice is 256 KB, more than the register file or the 227 KB of
// shared memory of one CTA, so the lo plane stays in registers and the hi plane lives in shared memory in fragment
// order (one conflict-free 16-byte load per thread and k-step);
// per step the only traffic is the h_t all-gather (forward) or the dh reduce-scatter (BPTT) inside the cluster through
// distributed shared memory.  It is point to point: every transfer completes the transaction count of one mbarrier of
// the receiving CTA per (buffer, source CTA), and a CTA waits for each source's data just before it uses it, so there
// is no per-step cluster barrier.  Batch is split across clusters (grid = C * ceil(B/NB)).
//   forward : D[gate rows(128) x NB] = W_slice[128 x H] * h_{s-1}^T           (swap-AB: M = gate rows)
//   backward: P[H x NB] = W_slice^T[H x 128] * dG_s^T  -> reduce-scatter of fp32 partials via DSMEM
// Tensor cores: mma.sync bf16, 3 passes (hi*hi, lo*hi, hi*lo), fp32 accumulate.
//
// Hand-off protocol (both kernels).  bar[buf][src] (arrival count 1) completes when this CTA has armed it with the
// byte count of one slice (arrive.expect_tx) and CTA `src` has delivered those bytes (complete_tx).  The data for step
// s >= 1 (forward) / iteration it >= 1 (BPTT) sits in buffer b = s & 1; buffer b is filled for the steps b+1, b+3,
// ..., so step s uses phase (s-1)/2 of bar[b][*] and waits on parity ((s-1) >> 1) & 1.  A barrier is armed once after
// init and re-armed by this CTA after all of its threads have passed the wait of the phase before (the __syncthreads
// that follows the waits), so it is never armed twice in one phase.
// Why no write-after-read hazard remains: CTA d writes step s+1's slice into my buffer b only after its own step-s
// MMAs (forward) / pointwise (BPTT) consumed the slice I sent at step s, and I send that slice only after a
// __syncthreads that follows my reads of buffer b at step s-1; a peer is therefore never more than one step ahead of
// the buffer it writes (BPTT: a peer sends its partials in m-tile groups, the first one right after its pointwise
// phase, so the chain is the same).  The same chain shows that the next phase of bar[b][d] cannot complete before
// every thread of mine has observed the current one, so parity waits are unambiguous.
// BPTT activation stage.  None of the BPTT's per-step global inputs (gates[s], cs[s], dh_head) depends on the
// recurrence, so each thread cp.asyncs step s-1's values for its own cells into stage[plane][n][unit] right after the
// pointwise phase of step s, and waits for them (cp.async.wait_group 0, no barrier: no thread reads a stage element
// another thread copied) at the top of the next pointwise phase; the pointwise phase then reads only shared memory.
// c_new (cs[s+1]) is c_prev of the step before and is carried in a register.
//  - stage write-after-read: a thread issues the next prefetch only after it has consumed the values it read from
//    the stage (they are in dgs before the __syncthreads that precedes the prefetch);
//  - in-place dG (dgates may alias gates): the thread that prefetches gates[s-1][b][q*H+u] is the only writer of
//    dgates[s-1][b][q*H+u], and it writes it only after its cp.async wait;
//  - repeat > 1: the keep / dgin accumulation is untouched.
// Every wait is bounded (wait_slice): on expiry it records a status word read by lstm_scan_error_status and carries on,
// so a protocol error is reported and the launch still ends.
#include <cooperative_groups.h>
#include <stdlib.h>

#include "gemm.cuh"
#include "lstm_scan.cuh"
#include "elementwise.cuh"
#include "sm90.cuh"

namespace cg = cooperative_groups;

namespace r2d2 {
namespace {

constexpr int SCAN_THREADS = 256;
constexpr int UNITS_PER_CTA = 32;
constexpr int ROWS_PER_CTA = 128;         // 4 gates x 32 units
constexpr int GT_LD = ROWS_PER_CTA + 4;   // fp32 gate tile [NB][132]: conflict-free fragment writes / unit reads
constexpr int DG_LD = ROWS_PER_CTA + 8;   // bf16 dG tile [NB][136]
constexpr unsigned long long kWaitLimitNs = 4000000000ull;

__device__ unsigned g_scan_status = 0;   // 1 = a bounded hand-off wait expired (sticky until read)

__device__ __forceinline__ float accurate_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

// waits until phase `parity` of `bar` has completed, for at most kWaitLimitNs; on expiry it sets g_scan_status and
// returns as if the data had arrived.  Once a wait has expired the run is lost and later waits do not stall it further.
__device__ __forceinline__ void wait_slice(uint64_t* bar, uint32_t parity) {
  if (sm90::mbar_try_wait(bar, parity)) return;
  if (*reinterpret_cast<volatile unsigned*>(&g_scan_status)) return;
  const unsigned long long t0 = global_ns();
  while (!sm90::mbar_try_wait(bar, parity)) {
    if (global_ns() - t0 > kWaitLimitNs) {
      atomicExch(&g_scan_status, 1u);
      return;
    }
  }
}

// phase parity of the hand-off barriers used at step (iteration) s >= 1: see the protocol note at the top
__device__ __forceinline__ uint32_t slice_parity(int s) { return (uint32_t)((s - 1) >> 1) & 1u; }

// ------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------
// W_hh hi plane in shared memory (H = 512): the register file cannot hold both planes of a 128 x 512 slice
template <int H> __host__ __device__ constexpr bool w_hi_in_smem() { return H > 256; }

template <int H, int NB>
struct FwdSmem {
  static constexpr int C = H / 32;
  static constexpr int HROW = UNITS_PER_CTA + 8;           // 80-byte rows: g * 20 words mod 32 are distinct, so the
                                                           // B-fragment loads are free of bank conflicts
  static constexpr int SLICE = 2 * NB * HROW;              // bf16 h_t slice of one source CTA [plane][n][unit]: one bulk copy
  static constexpr int W_BYTES = w_hi_in_smem<H>() ? (H / 16) * 8 * 32 * 16 : 0;   // hi fragments [ks][warp][lane][16 B]
  static constexpr int HB_ELEMS = 2 * C * SLICE;           // h operand [buf][src][plane][n][unit]
  static constexpr int GT_ELEMS = NB * GT_LD;              // fp32
  static constexpr int HS_ELEMS = SLICE;                   // bf16 staging of this CTA's slice
  static constexpr int BAR_OFF = W_BYTES + HB_ELEMS * 2 + GT_ELEMS * 4 + HS_ELEMS * 2;
  static constexpr int BYTES = BAR_OFF + 2 * C * 8;        // + mbarriers [buf][src]
  static_assert((SLICE * 2) % 16 == 0 && BAR_OFF % 16 == 0, "bulk copies need 16-byte granules");
  static_assert(BYTES <= 232448, "forward scan tile does not fit in 227 KB of shared memory");
};

template <int H, int NB>
__global__ void __launch_bounds__(SCAN_THREADS, 1) lstm_scan_fwd_kernel(ScanFwdParams p) {
  constexpr int C = H / 32, KS = H / 16, NT = NB / 8;
  constexpr bool WS = w_hi_in_smem<H>();
  using SM = FwdSmem<H, NB>;
  constexpr int HROW = SM::HROW, SLICE = SM::SLICE;
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int b0 = (blockIdx.x / C) * NB;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int g = lane >> 2, c = lane & 3;
  const int B = p.B, S = p.T * p.repeat;

  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint4* w_hi_s = reinterpret_cast<uint4*>(smem_raw);   // H = 512 only
  __nv_bfloat16* hb = reinterpret_cast<__nv_bfloat16*>(smem_raw + SM::W_BYTES);
  float* gt = reinterpret_cast<float*>(smem_raw + SM::W_BYTES + SM::HB_ELEMS * 2);
  __nv_bfloat16* hstage = reinterpret_cast<__nv_bfloat16*>(smem_raw + SM::W_BYTES + SM::HB_ELEMS * 2 + SM::GT_ELEMS * 4);
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem_raw + SM::BAR_OFF);   // [buf][src]

  // ---- initial state (before the weights, while few registers are live): full h0 tile -> hb[0]; own units -> hs[0], cs[0], c registers
  for (int idx = tid; idx < NB * H; idx += SCAN_THREADS) {
    const int n = idx / H, k = idx % H, b = b0 + n;
    float v = (b < B && p.h0) ? __ldg(p.h0 + (size_t)b * H + k) : 0.f;
    __nv_bfloat16 hi, lo;
    split_bf16(v, hi, lo);
    __nv_bfloat16* row = hb + (0 * C + k / UNITS_PER_CTA) * SLICE + n * HROW + k % UNITS_PER_CTA;
    row[0] = hi;
    row[NB * HROW] = lo;
  }
  const int ug = rank * 32 + lane;  // global hidden unit owned by this thread in the pointwise phase
  float cst[NT];
#pragma unroll
  for (int e = 0; e < NT; ++e) {
    const int b = b0 + w + 8 * e;
    cst[e] = 0.f;
    if (b < B) {
      float hv = p.h0 ? __ldg(p.h0 + (size_t)b * H + ug) : 0.f;
      float cv = p.c0 ? __ldg(p.c0 + (size_t)b * H + ug) : 0.f;
      p.hs[(size_t)b * H + ug] = hv;
      p.cs[(size_t)b * H + ug] = cv;
      cst[e] = cv;
    }
  }
  if (tid < 2 * C) {
    sm90::mbar_init(bar + tid, 1);
    sm90::fence_mbar_init_cluster();
    sm90::mbar_arrive_expect_tx(bar + tid, SLICE * 2);
  }

  // ---- W_hh slice -> resident A fragments (rows: local r = gate*32 + unit; warp w owns r in [16w,16w+16))
  uint32_t a_hi[WS ? 1 : KS][4], a_lo[KS][4];
  {
    const int gate = w >> 1;
    const int u_lo = (w & 1) * 16 + g;  // local unit of fragment row g; row g+8 -> unit u_lo+8
    const float* w_r0 = p.whh + (size_t)(gate * H + rank * 32 + u_lo) * H;
    const float* w_r1 = w_r0 + (size_t)8 * H;
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
      const int k = ks * 16 + 2 * c;
      float2 v0 = __ldg(reinterpret_cast<const float2*>(w_r0 + k));
      float2 v1 = __ldg(reinterpret_cast<const float2*>(w_r1 + k));
      float2 v2 = __ldg(reinterpret_cast<const float2*>(w_r0 + k + 8));
      float2 v3 = __ldg(reinterpret_cast<const float2*>(w_r1 + k + 8));
      uint32_t h[4];
      split_pack2(v0.x, v0.y, h[0], a_lo[ks][0]);
      split_pack2(v1.x, v1.y, h[1], a_lo[ks][1]);
      split_pack2(v2.x, v2.y, h[2], a_lo[ks][2]);
      split_pack2(v3.x, v3.y, h[3], a_lo[ks][3]);
      if constexpr (WS) {
        w_hi_s[(ks * 8 + w) * 32 + lane] = make_uint4(h[0], h[1], h[2], h[3]);
      } else {
#pragma unroll
        for (int f = 0; f < 4; ++f) a_hi[ks][f] = h[f];
      }
    }
  }
  __syncthreads();
  cluster.sync();  // every CTA of the cluster has started and armed its barriers: remote transfers may start

  const size_t gstride = (size_t)4 * H;
  for (int s = 0; s < S; ++s) {
    const int cur = s & 1, nxt = cur ^ 1;
    const int t = s / p.repeat;

    // this step's input projection -> the gate tile, for the elements whose MMA fragment this thread adds below:
    // the copies run behind the MMAs without holding registers (gates may alias gin: each element is read here
    // before the pointwise phase of this step overwrites it)
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int f = 0; f < 4; ++f) {
        const int n = nt * 8 + 2 * c + (f & 1), r = 16 * w + g + (f >> 1) * 8, b = b0 + n;
        if (b < B) sm90::cp_async_4(gt + n * GT_LD + r, p.gin + ((size_t)t * B + b) * gstride + (r >> 5) * H + rank * 32 + (r & 31));
      }
    sm90::cp_async_commit();

    // ---- tensor-core part: acc[128 x NB] = W_slice * h_{s-1}^T
    float acc[NT][4];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[nt][e] = 0.f;
    const __nv_bfloat16* hb_cur = hb + cur * C * SLICE;
    uint64_t* bar_cur = bar + cur * C;
    const uint32_t parity = slice_parity(s);
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
      // k-steps 2d, 2d+1 read the slice of source CTA d: wait for it here, so that the MMAs on the slices that
      // arrived first overlap the arrival of the later ones (step 0 reads h0, written by this CTA)
      if ((ks & 1) == 0 && s > 0) wait_slice(bar_cur + ks / 2, parity);
      const __nv_bfloat16* hb_hi = hb_cur + (ks / 2) * SLICE;
      const __nv_bfloat16* hb_lo = hb_hi + NB * HROW;
      uint32_t ah[4];
      if constexpr (WS) {
        const uint4 v = w_hi_s[(ks * 8 + w) * 32 + lane];
        ah[0] = v.x; ah[1] = v.y; ah[2] = v.z; ah[3] = v.w;
      } else {
#pragma unroll
        for (int f = 0; f < 4; ++f) ah[f] = a_hi[ks][f];
      }
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        const int off = (nt * 8 + g) * HROW + (ks & 1) * 16 + 2 * c;
        uint32_t bh[2], bl[2];
        bh[0] = *reinterpret_cast<const uint32_t*>(hb_hi + off);
        bh[1] = *reinterpret_cast<const uint32_t*>(hb_hi + off + 8);
        bl[0] = *reinterpret_cast<const uint32_t*>(hb_lo + off);
        bl[1] = *reinterpret_cast<const uint32_t*>(hb_lo + off + 8);
        mma_bf16_16816(acc[nt], a_lo[ks], bh);
        mma_bf16_16816(acc[nt], ah, bl);
        mma_bf16_16816(acc[nt], ah, bh);
      }
    }
    // fragment + input projection -> gate tile gt[n][local row] (rows b >= B hold garbage and are never read)
    sm90::cp_async_wait_all();
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      const int n = nt * 8 + 2 * c, r = 16 * w + g;
      gt[n * GT_LD + r] += acc[nt][0];
      gt[(n + 1) * GT_LD + r] += acc[nt][1];
      gt[n * GT_LD + r + 8] += acc[nt][2];
      gt[(n + 1) * GT_LD + r + 8] += acc[nt][3];
    }
    if (w == 0 && lane < C) sm90::bulk_wait_read_all();   // last step's sends have read hstage
    __syncthreads();
    // every thread has passed its waits on bar[cur][*]: arm them for the step after next
    if (s > 0 && tid < C) sm90::mbar_arrive_expect_tx(bar_cur + tid, SLICE * 2);

    // ---- pointwise LSTM cell: thread = (unit = lane, batch column n = w + 8e); coalesced along units
#pragma unroll
    for (int e = 0; e < NT; ++e) {
      const int n = w + 8 * e, b = b0 + n;
      __nv_bfloat16 hi = __float2bfloat16_rn(0.f), lo = hi;
      if (b < B) {
        const float* gr = gt + n * GT_LD + lane;
        const float ig = accurate_sigmoid(gr[0]);
        const float fg = accurate_sigmoid(gr[32]);
        const float gg = tanhf(gr[64]);
        const float og = accurate_sigmoid(gr[96]);
        const float cn = fg * cst[e] + ig * gg;
        const float hn = og * tanhf(cn);
        cst[e] = cn;
        if (!p.no_save) {   // gates and c are read by the BPTT only
          float* go = p.gates + ((size_t)s * B + b) * gstride + ug;
          go[0] = ig; go[H] = fg; go[2 * H] = gg; go[3 * H] = og;
          p.cs[((size_t)(s + 1) * B + b) * H + ug] = cn;
        }
        p.hs[((size_t)(s + 1) * B + b) * H + ug] = hn;
        if (p.head_in && (s % p.repeat) == p.repeat - 1)
          p.head_in[((size_t)t * B + b) * H + ug] = tanhf(hn);
        split_bf16(hn, hi, lo);
      }
      hstage[(0 * NB + n) * HROW + lane] = hi;
      hstage[(1 * NB + n) * HROW + lane] = lo;
    }
    sm90::fence_proxy_async_smem();   // the bulk copies below read hstage through the async proxy
    __syncthreads();

    // ---- all-gather of h_s inside the cluster: one bulk copy of this CTA's slice into every CTA's next operand
    // buffer, completing that CTA's bar[nxt][rank]
    if (s + 1 < S && w == 0 && lane < C) {
      const uint32_t slot = sm90::smem_u32(hb + (nxt * C + rank) * SLICE);
      const uint32_t slot_bar = sm90::smem_u32(bar + nxt * C + rank);
      sm90::bulk_copy_s2cluster(sm90::map_cluster(slot, lane), sm90::smem_u32(hstage), SLICE * 2,
                                sm90::map_cluster(slot_bar, lane));
      sm90::bulk_commit();
    }
  }
  cluster.sync();   // no CTA leaves while a peer may still deliver into its shared memory
}

// ------------------------------------------------------------------------------------------------
// backward (BPTT)
// ------------------------------------------------------------------------------------------------
template <int H, int NB>
struct BwdSmem {
  static constexpr int C = H / 32;
  static constexpr int DG_ELEMS = 2 * NB * DG_LD;               // bf16 [plane][n][local gate row]
  static constexpr int PS_LD = NB + 2;                          // 2-way instead of 16-way bank conflicts on the unit-strided reads
  static constexpr int PS_ELEMS = 2 * C * UNITS_PER_CTA * PS_LD; // fp32 [buf][src rank][unit][n]
  static constexpr int PS_BYTES_PER_SRC = UNITS_PER_CTA * NB * 4; // delivered per (buf, src): the pad columns stay unwritten
  static constexpr int MT = (H / 16 + 7) / 8;
  static constexpr int W_BYTES = w_hi_in_smem<H>() ? MT * 8 * 8 * 32 * 16 : 0;   // hi fragments [i][ks][warp][lane][16 B]
  static constexpr int STAGE_PLANES = 6;                        // gates i, f, g, o; c_prev; dh_head
  static constexpr int STAGE_ELEMS = STAGE_PLANES * NB * UNITS_PER_CTA;   // fp32 [plane][n][unit], one step
  static constexpr int BAR_OFF = W_BYTES + DG_ELEMS * 2 + PS_ELEMS * 4 + STAGE_ELEMS * 4;
  static constexpr int BYTES = BAR_OFF + 2 * C * 8;              // + mbarriers [buf][src]
  static_assert(BAR_OFF % 8 == 0, "mbarrier alignment");
  static_assert(BYTES <= 232448, "BPTT scan tile does not fit in 227 KB of shared memory");
};

template <int H, int NB>
__global__ void __launch_bounds__(SCAN_THREADS, 1) lstm_scan_bwd_kernel(ScanBwdParams p) {
  constexpr int C = H / 32, NT = NB / 8;
  constexpr int M_TILES = H / 16;
  constexpr int MT = (M_TILES + 7) / 8;  // m-tiles per warp
  constexpr int KS = ROWS_PER_CTA / 16;  // 8
  constexpr bool WS = w_hi_in_smem<H>();
  // m-tiles per reduce-scatter group: at H = 512 each m-tile's partials leave as soon as they are final; below, a warp
  // has at most two m-tiles and one group measured faster
  constexpr int MG = WS ? 1 : MT;
  using SM = BwdSmem<H, NB>;
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int b0 = (blockIdx.x / C) * NB;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int g = lane >> 2, c = lane & 3;
  const int B = p.B, S = p.T * p.repeat;

  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint4* w_hi_s = reinterpret_cast<uint4*>(smem_raw);   // H = 512 only
  __nv_bfloat16* dgs = reinterpret_cast<__nv_bfloat16*>(smem_raw + SM::W_BYTES);
  float* ps = reinterpret_cast<float*>(smem_raw + SM::W_BYTES + SM::DG_ELEMS * 2);
  float* stage = ps + SM::PS_ELEMS;                                       // [plane][n][unit]
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem_raw + SM::BAR_OFF);   // [buf][src]
  constexpr int PLANE = NB * UNITS_PER_CTA;
  constexpr size_t gstride = (size_t)4 * H;

  // step s adds dh_head row (s - head_first_step) / repeat when it is the last repeat of a head row
  auto head_step = [&](int s) {
    const int rel = s - p.head_first_step;
    return p.dh_head && rel >= 0 && (rel % p.repeat) == p.repeat - 1;
  };
  // gates, c_prev (and dh_head on head steps) of step s for exactly the cells this thread processes in the pointwise
  // phase -> stage; the copies land while the MMAs, the reduce-scatter and the dh waits of the step before run.
  // The addresses are rebuilt from %tid.x at every call: kept live instead, they would cost registers through the W_hh
  // prologue below, which at H = 512 already runs at the 255-register limit.
  auto prefetch = [&](int s) {
    const int rel = s - p.head_first_step;
    const bool head = head_step(s);
    unsigned tv;
    asm volatile("mov.u32 %0, %%tid.x;" : "=r"(tv));   // volatile: not hoisted out of the step loop
    const int lane = tv & 31, w = tv >> 5, ug = rank * 32 + lane;
#pragma unroll
    for (int e = 0; e < NT; ++e) {
      const int n = w + 8 * e, b = b0 + n;
      if (b < B) {
        float* st = stage + n * UNITS_PER_CTA + lane;
        const float* gs = p.gates + ((size_t)s * B + b) * gstride + ug;
#pragma unroll
        for (int q = 0; q < 4; ++q) sm90::cp_async_4(st + q * PLANE, gs + q * H);
        sm90::cp_async_4(st + 4 * PLANE, p.cs + ((size_t)s * B + b) * H + ug);
        if (head) sm90::cp_async_4(st + 5 * PLANE, p.dh_head + ((size_t)(rel / p.repeat) * B + b) * H + ug);
      }
    }
    sm90::cp_async_commit();
  };

  if (tid < 2 * C) {
    sm90::mbar_init(bar + tid, 1);
    sm90::fence_mbar_init_cluster();
    sm90::mbar_arrive_expect_tx(bar + tid, SM::PS_BYTES_PER_SRC);
  }
  prefetch(S - 1);   // overlaps the W_hh prologue below

  // ---- W_hh slice (transposed use): A(m = j output unit, k = local gate row r) = W_hh[grow(r)][j]
  // element (j, r) with j = mi * 16 + g + (f & 1) * 8, r = ks * 16 + 2c + (f >> 1) * 8 (local gate rows r, r+1: gate
  // r / 32 = ks / 2, unit r % 32) sits at a compile-time offset from one per-thread pointer, so the unrolled loads
  // need no further address registers (and spill less at H = 512)
  const float* w_t = p.whh + (size_t)(rank * 32 + 2 * c) * H + w * MT * 16 + g;
  uint32_t a_hi[WS ? 1 : MT][WS ? 1 : KS][4], a_lo[MT][KS][4];
#pragma unroll
  for (int i = 0; i < MT; ++i) {
    const int mi = w * MT + i;
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
      uint32_t h[4];
#pragma unroll
      for (int f = 0; f < 4; ++f) {
        float v0 = 0.f, v1 = 0.f;
        if (mi < M_TILES) {
          const float* w0 = w_t + ((ks >> 1) * H + (ks & 1) * 16 + (f >> 1) * 8) * H + i * 16 + (f & 1) * 8;
          v0 = __ldg(w0);
          v1 = __ldg(w0 + H);  // r even -> r+1 stays in the same gate block
        }
        split_pack2(v0, v1, h[f], a_lo[i][ks][f]);
      }
      if constexpr (WS) {
        w_hi_s[((i * KS + ks) * 8 + w) * 32 + lane] = make_uint4(h[0], h[1], h[2], h[3]);
      } else {
#pragma unroll
        for (int f = 0; f < 4; ++f) a_hi[i][ks][f] = h[f];
      }
    }
  }

  __syncthreads();   // W_hh hi fragments in shared memory (H = 512) before the first MMA
  const int ug = rank * 32 + lane;
  // c_new of the cell at step s (cs[s+1]) is c_prev of step s+1: it stays in a register, only cs[S] is loaded here
  float dcn[NT], keep[NT][4], c_new[NT];
#pragma unroll
  for (int e = 0; e < NT; ++e) {
    const int b = b0 + w + 8 * e;
    dcn[e] = 0.f;
    c_new[e] = b < B ? __ldg(p.cs + ((size_t)S * B + b) * H + ug) : 0.f;
#pragma unroll
    for (int q = 0; q < 4; ++q) keep[e][q] = 0.f;
  }
  cluster.sync();

  for (int it = 0; it < S; ++it) {
    const int s = S - 1 - it;
    const int buf = it & 1;
    const int t = s / p.repeat;
    const bool has_head = head_step(s);

    // partial dh from every source CTA (iteration 0 has none), added in source order 0..C-1 as each one arrives
    float dh_rec[NT];
#pragma unroll
    for (int e = 0; e < NT; ++e) dh_rec[e] = 0.f;
    if (it > 0) {
      const uint32_t parity = slice_parity(it);
#pragma unroll
      for (int src = 0; src < C; ++src) {
        wait_slice(bar + buf * C + src, parity);
        const float* pr = ps + ((buf * C + src) * UNITS_PER_CTA + lane) * SM::PS_LD + w;
#pragma unroll
        for (int e = 0; e < NT; ++e) dh_rec[e] += pr[8 * e];
      }
    }
    sm90::cp_async_wait_all();   // this step's stage, copied by this thread one iteration earlier

    // ---- pointwise backward of the cell (thread = (unit = lane, n = w + 8e))
#pragma unroll
    for (int e = 0; e < NT; ++e) {
      const int n = w + 8 * e, b = b0 + n;
      float dg[4] = {0.f, 0.f, 0.f, 0.f};
      if (b < B) {
        const float* st = stage + n * UNITS_PER_CTA + lane;
        float dh = dh_rec[e];
        if (has_head) dh += st[5 * PLANE];
        const float ig = st[0], fg = st[PLANE], gg = st[2 * PLANE], og = st[3 * PLANE];
        const float c_prev = st[4 * PLANE];
        const float tc = tanhf(c_new[e]);
        c_new[e] = c_prev;
        const float dc = dcn[e] + dh * og * (1.f - tc * tc);
        dg[3] = dh * tc * og * (1.f - og);
        dg[0] = dc * gg * ig * (1.f - ig);
        dg[1] = dc * c_prev * fg * (1.f - fg);
        dg[2] = dc * ig * (1.f - gg * gg);
        dcn[e] = dc * fg;
        float* go = p.dgates + ((size_t)s * B + b) * gstride + ug;
        go[0] = dg[0]; go[H] = dg[1]; go[2 * H] = dg[2]; go[3 * H] = dg[3];
        if (p.repeat > 1) {
#pragma unroll
          for (int q = 0; q < 4; ++q) keep[e][q] += dg[q];
          if (s % p.repeat == 0) {
            float* gi = p.dgin + ((size_t)t * B + b) * gstride + ug;
#pragma unroll
            for (int q = 0; q < 4; ++q) { gi[q * H] = keep[e][q]; keep[e][q] = 0.f; }
          }
        }
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        __nv_bfloat16 hi, lo;
        split_bf16(dg[q], hi, lo);
        dgs[(0 * NB + n) * DG_LD + q * 32 + lane] = hi;
        dgs[(1 * NB + n) * DG_LD + q * 32 + lane] = lo;
      }
    }
    __syncthreads();
    // every thread has passed its waits on bar[buf][*]: arm them for the iteration after next
    if (it > 0 && tid < C) sm90::mbar_arrive_expect_tx(bar + buf * C + tid, SM::PS_BYTES_PER_SRC);

    if (s > 0) {
      prefetch(s - 1);
      // ---- partial dh_{s-1}[j, n] over this CTA's 128 gate rows, MG m-tiles at a time: a group's partials leave by
      // st.async as soon as its last k-step is done, so the reduce-scatter overlaps the next group's MMAs.  Every
      // accumulator sees the same MMAs in the same k order as with one group; the dG fragments are re-read per group.
      const __nv_bfloat16* d_hi = dgs;
      const __nv_bfloat16* d_lo = dgs + NB * DG_LD;
      const uint32_t slot_bar = sm90::smem_u32(bar + (buf ^ 1) * C + rank);
#pragma unroll
      for (int i0 = 0; i0 < MT; i0 += MG) {
        float acc[MG][NT][4];
#pragma unroll
        for (int i = 0; i < MG; ++i)
#pragma unroll
          for (int nt = 0; nt < NT; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[i][nt][e] = 0.f;
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
          uint32_t bh[NT][2], bl[NT][2];
#pragma unroll
          for (int nt = 0; nt < NT; ++nt) {
            const int off = (nt * 8 + g) * DG_LD + ks * 16 + 2 * c;
            bh[nt][0] = *reinterpret_cast<const uint32_t*>(d_hi + off);
            bh[nt][1] = *reinterpret_cast<const uint32_t*>(d_hi + off + 8);
            bl[nt][0] = *reinterpret_cast<const uint32_t*>(d_lo + off);
            bl[nt][1] = *reinterpret_cast<const uint32_t*>(d_lo + off + 8);
          }
#pragma unroll
          for (int i = 0; i < MG; ++i) {
            uint32_t ah[4];
            if constexpr (WS) {
              const uint4 v = w_hi_s[(((i0 + i) * KS + ks) * 8 + w) * 32 + lane];
              ah[0] = v.x; ah[1] = v.y; ah[2] = v.z; ah[3] = v.w;
            } else {
#pragma unroll
              for (int f = 0; f < 4; ++f) ah[f] = a_hi[i0 + i][ks][f];
            }
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) {
              mma_bf16_16816(acc[i][nt], a_lo[i0 + i][ks], bh[nt]);
              mma_bf16_16816(acc[i][nt], ah, bl[nt]);
              mma_bf16_16816(acc[i][nt], ah, bh[nt]);
            }
          }
        }
        // ---- reduce-scatter: partial rows j go to the CTA that owns unit j (slot = my rank), fp32 st.async into its
        // shared memory, each store completing its bytes on the owner's bar[buf ^ 1][rank]
#pragma unroll
        for (int i = 0; i < MG; ++i) {
          const int mi = w * MT + i0 + i;
          if (mi < M_TILES) {
#pragma unroll
            for (int h2 = 0; h2 < 2; ++h2) {
              const int j = mi * 16 + g + h2 * 8;
              const int owner = j >> 5, jl = j & 31;
              const uint32_t slot = sm90::map_cluster(
                  sm90::smem_u32(ps + (((buf ^ 1) * C + rank) * UNITS_PER_CTA + jl) * SM::PS_LD), owner);
              const uint32_t owner_bar = sm90::map_cluster(slot_bar, owner);
#pragma unroll
              for (int nt = 0; nt < NT; ++nt)
                sm90::st_async_f2(slot + (nt * 8 + 2 * c) * 4, acc[i][nt][2 * h2], acc[i][nt][2 * h2 + 1], owner_bar);
            }
          }
        }
      }
    }
    __syncthreads();   // dgs is rewritten by the next iteration's pointwise phase
  }
  cluster.sync();   // no CTA leaves while a peer may still deliver into its shared memory
}

// ------------------------------------------------------------------------------------------------
// per-step path (any H): one GEMM + one pointwise kernel per step.  Correct for every size; used when the cluster
// kernels do not cover H (H not a multiple of 32 in 32..512) and as the A/B reference (lstm_scan_set_impl(0)).
// ------------------------------------------------------------------------------------------------
__global__ void lstm_cell_fwd_pointwise(const float* __restrict__ gpre, const float* __restrict__ c_prev,
                                        float* __restrict__ gates, float* __restrict__ h_out,
                                        float* __restrict__ c_out, float* __restrict__ head_in, int B, int H) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * H) return;
  const int b = idx / H, u = idx % H;
  const float* gr = gpre + (size_t)b * 4 * H + u;
  const float ig = accurate_sigmoid(gr[0]), fg = accurate_sigmoid(gr[H]);
  const float gg = tanhf(gr[2 * H]), og = accurate_sigmoid(gr[3 * H]);
  const float cn = fg * c_prev[idx] + ig * gg;
  const float hn = og * tanhf(cn);
  float* go = gates + (size_t)b * 4 * H + u;
  go[0] = ig; go[H] = fg; go[2 * H] = gg; go[3 * H] = og;
  h_out[idx] = hn;
  c_out[idx] = cn;
  if (head_in) head_in[idx] = tanhf(hn);
}

__global__ void lstm_cell_bwd_pointwise(const float* __restrict__ gates, const float* __restrict__ c_prev,
                                        const float* __restrict__ c_new, const float* __restrict__ dh_head,
                                        const float* __restrict__ dh_rec, float* __restrict__ dc_state,
                                        float* __restrict__ dgates, float* __restrict__ dgin, int dgin_mode,
                                        int B, int H) {
  // dgin_mode: 0 = none, 1 = overwrite (first visit of this input row), 2 = accumulate
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * H) return;
  const int b = idx / H, u = idx % H;
  const float* gs = gates + (size_t)b * 4 * H + u;
  const float ig = gs[0], fg = gs[H], gg = gs[2 * H], og = gs[3 * H];
  float dh = dh_rec ? dh_rec[idx] : 0.f;
  if (dh_head) dh += dh_head[idx];
  const float tc = tanhf(c_new[idx]);
  const float dc = dc_state[idx] + dh * og * (1.f - tc * tc);
  float dg[4];
  dg[3] = dh * tc * og * (1.f - og);
  dg[0] = dc * gg * ig * (1.f - ig);
  dg[1] = dc * c_prev[idx] * fg * (1.f - fg);
  dg[2] = dc * ig * (1.f - gg * gg);
  dc_state[idx] = dc * fg;
  float* go = dgates + (size_t)b * 4 * H + u;
  float* gi = dgin ? dgin + (size_t)b * 4 * H + u : nullptr;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    go[q * H] = dg[q];
    if (dgin_mode == 1) gi[q * H] = dg[q];
    else if (dgin_mode == 2) gi[q * H] += dg[q];
  }
}

int scan_forward_generic(const ScanFwdParams& p, float* scratch, cudaStream_t stream) {
  const int B = p.B, H = p.H, S = p.T * p.repeat;
  const size_t bh = (size_t)B * H;
  R2D2_REQUIRE(scratch != nullptr, "generic scan needs scratch");
  if (p.h0) R2D2_CUDA_TRY(cudaMemcpyAsync(p.hs, p.h0, bh * 4, cudaMemcpyDeviceToDevice, stream));
  else R2D2_CUDA_TRY(cudaMemsetAsync(p.hs, 0, bh * 4, stream));
  if (p.c0) R2D2_CUDA_TRY(cudaMemcpyAsync(p.cs, p.c0, bh * 4, cudaMemcpyDeviceToDevice, stream));
  else R2D2_CUDA_TRY(cudaMemsetAsync(p.cs, 0, bh * 4, stream));
  const int blocks = ceil_div((int)bh, 256);
  for (int s = 0; s < S; ++s) {
    const int t = s / p.repeat;
    GemmParams g;
    g.A = p.hs + (size_t)s * bh; g.lda = H;
    g.B = p.whh; g.ldb = H;
    g.C = scratch; g.ldc = 4 * H;
    g.M = B; g.N = 4 * H; g.K = H;
    g.Z = p.gin + (size_t)t * B * 4 * H; g.ldz = 4 * H;
    g.epilogue = EPI_ADD_Z;
    R2D2_TRY(gemm_f32(g, GEMM_NT, stream));
    float* head = (p.head_in && (s % p.repeat) == p.repeat - 1) ? p.head_in + (size_t)t * bh : nullptr;
    lstm_cell_fwd_pointwise<<<blocks, 256, 0, stream>>>(scratch, p.cs + (size_t)s * bh,
                                                         p.gates + (size_t)s * B * 4 * H, p.hs + (size_t)(s + 1) * bh,
                                                         p.cs + (size_t)(s + 1) * bh, head, B, H);
    count_launch();
  }
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

int scan_backward_generic(const ScanBwdParams& p, cudaStream_t stream) {
  const int B = p.B, H = p.H, S = p.T * p.repeat;
  const size_t bh = (size_t)B * H;
  R2D2_REQUIRE(p.scratch != nullptr, "generic scan needs scratch");
  float* dh_rec = p.scratch;
  float* dc_state = p.scratch + bh;
  R2D2_CUDA_TRY(cudaMemsetAsync(p.scratch, 0, 2 * bh * 4, stream));
  const int blocks = ceil_div((int)bh, 256);
  for (int s = S - 1; s >= 0; --s) {
    const int t = s / p.repeat;
    const int rel = s - p.head_first_step;
    const bool has_head = p.dh_head && rel >= 0 && (rel % p.repeat) == p.repeat - 1;
    const float* head = has_head ? p.dh_head + (size_t)(rel / p.repeat) * bh : nullptr;
    int mode = 0;
    if (p.repeat > 1) mode = ((s % p.repeat) == p.repeat - 1) ? 1 : 2;
    lstm_cell_bwd_pointwise<<<blocks, 256, 0, stream>>>(
        p.gates + (size_t)s * B * 4 * H, p.cs + (size_t)s * bh, p.cs + (size_t)(s + 1) * bh, head,
        (s == S - 1) ? nullptr : dh_rec, dc_state, p.dgates + (size_t)s * B * 4 * H,
        mode ? p.dgin + (size_t)t * B * 4 * H : nullptr, mode, B, H);
    count_launch();
    if (s > 0) {
      GemmParams g;
      g.A = p.dgates + (size_t)s * B * 4 * H; g.lda = 4 * H;
      g.B = p.whh; g.ldb = H;
      g.C = dh_rec; g.ldc = H;
      g.M = B; g.N = H; g.K = 4 * H;
      R2D2_TRY(gemm_f32(g, GEMM_NN, stream));
    }
  }
  R2D2_CUDA_TRY(cudaGetLastError());
  return R2D2_OK;
}

template <typename Kern>
int set_cluster_attributes(Kern kern, int cluster_size, int smem_bytes) {
  R2D2_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
  if (cluster_size > 8) R2D2_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
  return R2D2_OK;
}

cudaLaunchConfig_t cluster_config(int cluster_size, int n_clusters, int smem_bytes, cudaStream_t stream,
                                  cudaLaunchAttribute* attr) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(cluster_size * n_clusters);
  cfg.blockDim = dim3(SCAN_THREADS);
  cfg.dynamicSmemBytes = smem_bytes;
  cfg.stream = stream;
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cluster_size;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cfg;
}

template <typename Kern, typename Params>
int launch_cluster(Kern kern, const Params& p, int cluster_size, int n_clusters, int smem_bytes, cudaStream_t stream) {
  R2D2_TRY(set_cluster_attributes(kern, cluster_size, smem_bytes));
  cudaLaunchAttribute attr[1];
  cudaLaunchConfig_t cfg = cluster_config(cluster_size, n_clusters, smem_bytes, stream, attr);
  R2D2_CUDA_TRY(cudaLaunchKernelEx(&cfg, kern, p));
  count_launch();
  return R2D2_OK;
}

// clusters of this kernel the device keeps resident at once (GPC geometry decides, not the SM count alone)
template <typename Kern>
int resident_clusters(Kern kern, int cluster_size, int smem_bytes, int* out) {
  R2D2_TRY(set_cluster_attributes(kern, cluster_size, smem_bytes));
  cudaLaunchAttribute attr[1];
  cudaLaunchConfig_t cfg = cluster_config(cluster_size, 1, smem_bytes, nullptr, attr);
  R2D2_CUDA_TRY(cudaOccupancyMaxActiveClusters(out, kern, &cfg));
  return R2D2_OK;
}

// Batch columns per cluster: the smallest tile whose clusters are all resident in one wave (per-step cost is
// dominated by fixed latencies, so more, narrower clusters win as long as they are co-resident); the widest tile
// that fits in shared memory otherwise (32 rows up to H = 256, 16 at H = 512).
template <int H, typename K8, typename K16, typename K32>
int pick_nb(int B, K8 k8, int smem8, K16 k16, int smem16, K32 k32, int smem32, int* nb) {
  int fit = 0;
  R2D2_TRY(resident_clusters(k8, H / 32, smem8, &fit));
  if (ceil_div(B, 8) <= fit) { *nb = 8; return R2D2_OK; }
  R2D2_TRY(resident_clusters(k16, H / 32, smem16, &fit));
  if (ceil_div(B, 16) <= fit || !k32) { *nb = 16; return R2D2_OK; }
  *nb = 32;
  (void)smem32;
  return R2D2_OK;
}

template <int H>
int fwd_dispatch(const ScanFwdParams& p, cudaStream_t stream) {
  constexpr bool WIDE = !w_hi_in_smem<H>();   // a 32-row tile fits next to the weights only below H = 512
  constexpr int NB3 = WIDE ? 32 : 16;
  int nb = 0;
  R2D2_TRY(pick_nb<H>(p.B, lstm_scan_fwd_kernel<H, 8>, FwdSmem<H, 8>::BYTES, lstm_scan_fwd_kernel<H, 16>,
                      FwdSmem<H, 16>::BYTES, WIDE ? lstm_scan_fwd_kernel<H, NB3> : nullptr, FwdSmem<H, NB3>::BYTES, &nb));
  if (nb == 8)
    return launch_cluster(lstm_scan_fwd_kernel<H, 8>, p, H / 32, ceil_div(p.B, 8), FwdSmem<H, 8>::BYTES, stream);
  if (nb == 16)
    return launch_cluster(lstm_scan_fwd_kernel<H, 16>, p, H / 32, ceil_div(p.B, 16), FwdSmem<H, 16>::BYTES, stream);
  return launch_cluster(lstm_scan_fwd_kernel<H, NB3>, p, H / 32, ceil_div(p.B, NB3), FwdSmem<H, NB3>::BYTES, stream);
}
template <int H>
int bwd_dispatch(const ScanBwdParams& p, cudaStream_t stream) {
  constexpr bool WIDE = !w_hi_in_smem<H>();
  constexpr int NB3 = WIDE ? 32 : 16;
  int nb = 0;
  R2D2_TRY(pick_nb<H>(p.B, lstm_scan_bwd_kernel<H, 8>, BwdSmem<H, 8>::BYTES, lstm_scan_bwd_kernel<H, 16>,
                      BwdSmem<H, 16>::BYTES, WIDE ? lstm_scan_bwd_kernel<H, NB3> : nullptr, BwdSmem<H, NB3>::BYTES, &nb));
  if (nb == 8)
    return launch_cluster(lstm_scan_bwd_kernel<H, 8>, p, H / 32, ceil_div(p.B, 8), BwdSmem<H, 8>::BYTES, stream);
  if (nb == 16)
    return launch_cluster(lstm_scan_bwd_kernel<H, 16>, p, H / 32, ceil_div(p.B, 16), BwdSmem<H, 16>::BYTES, stream);
  return launch_cluster(lstm_scan_bwd_kernel<H, NB3>, p, H / 32, ceil_div(p.B, NB3), BwdSmem<H, NB3>::BYTES, stream);
}

}  // namespace

bool lstm_scan_cluster_supported(int H) { return H == 32 || H == 64 || H == 128 || H == 256 || H == 512; }

static int g_scan_impl = -1;
void lstm_scan_set_impl(int impl) { g_scan_impl = impl ? 1 : 0; }
int lstm_scan_get_impl() {
  if (g_scan_impl < 0) {
    const char* e = getenv("R2D2_SCAN_IMPL");
    g_scan_impl = (e && (e[0] == 's' || e[0] == '0')) ? 0 : 1;
  }
  return g_scan_impl;
}
static bool use_cluster_kernels(int H) { return lstm_scan_cluster_supported(H) && lstm_scan_get_impl() == 1; }

int lstm_scan_error_status(int* out, cudaStream_t stream) {
  R2D2_REQUIRE(out, "null");
  unsigned v = 0;
  R2D2_CUDA_TRY(cudaMemcpyFromSymbolAsync(&v, g_scan_status, sizeof(v), 0, cudaMemcpyDeviceToHost, stream));
  R2D2_CUDA_TRY(cudaStreamSynchronize(stream));
  *out = (int)v;
  return R2D2_OK;
}

// the per-step path can be selected for every hidden size (lstm_scan_set_impl(0)), so its scratch is always reserved
size_t lstm_scan_fwd_scratch_floats(int B, int H) { return (size_t)B * 4 * H; }
size_t lstm_scan_bwd_scratch_floats(int B, int H) { return (size_t)2 * B * H; }

int lstm_scan_forward(const ScanFwdParams& p, cudaStream_t stream) {
  R2D2_REQUIRE(p.gin && p.whh && p.gates && p.hs && p.cs, "null pointer");
  R2D2_REQUIRE(p.T > 0 && p.B > 0 && p.H > 0 && p.repeat >= 1, "shape");
  R2D2_REQUIRE(p.repeat == 1 || p.gates != p.gin, "gates must not alias gin when repeat > 1");
  if (use_cluster_kernels(p.H)) {
    switch (p.H) {
      case 32: return fwd_dispatch<32>(p, stream);
      case 64: return fwd_dispatch<64>(p, stream);
      case 128: return fwd_dispatch<128>(p, stream);
      case 256: return fwd_dispatch<256>(p, stream);
      case 512: return fwd_dispatch<512>(p, stream);
      default: break;
    }
  }
  return scan_forward_generic(p, p.scratch, stream);
}

int lstm_scan_backward(const ScanBwdParams& p, cudaStream_t stream) {
  R2D2_REQUIRE(p.gates && p.hs && p.cs && p.whh && p.dgates, "null pointer");
  R2D2_REQUIRE(p.T > 0 && p.B > 0 && p.H > 0 && p.repeat >= 1, "shape");
  R2D2_REQUIRE(p.repeat == 1 || (p.dgin && p.dgin != p.dgates), "dgin buffer required when repeat > 1");
  int rc = R2D2_OK;
  switch (use_cluster_kernels(p.H) ? p.H : 0) {
    case 32: rc = bwd_dispatch<32>(p, stream); break;
    case 64: rc = bwd_dispatch<64>(p, stream); break;
    case 128: rc = bwd_dispatch<128>(p, stream); break;
    case 256: rc = bwd_dispatch<256>(p, stream); break;
    case 512: rc = bwd_dispatch<512>(p, stream); break;
    default: rc = scan_backward_generic(p, stream); break;
  }
  R2D2_TRY(rc);
  if (p.dbias) {  // sum_t dgin_t == sum_s dgates_s
    const float* src = p.repeat > 1 ? p.dgin : p.dgates;
    R2D2_TRY(colsum(src, 4 * p.H, p.T * p.B, 4 * p.H, p.dbias, p.dbias2, stream));
  }
  return R2D2_OK;
}

}  // namespace r2d2

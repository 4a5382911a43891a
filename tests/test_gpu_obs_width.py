"""Observation widths on the GPU: every kernel route that is chosen by the observation size O, checked against float64
and the CPU port of the reference.

 1. The actor's l1, z1 = tanh(obs W1^T + b1), through r2d2_gemm_f32: an NT product with K = O and one K segment.  O <= 32
    runs thin_smallk_kernel, 33 <= O <= 63 the mma.sync kernel, O >= 64 wgmma unless fewer than 32 rows (mma.sync).
 2. Actor and critic chains through r2d2_lstm_net_forward / _backward at O in every bucket, H in {32, 64, 128, 512} and
    T·B = 515 (and 21) rows, against oracle/learner_oracle.py.  The obs block of dW1 (TN, M = H, N = O, K = T·B, db1
    fused as a column sum) runs thin_tn_kernel<Q> or the wide kernels; at H = 32 <= O the narrow side is the M side
    (small_is_m) and db1 comes from the narrow-side column sum.  l1.weight's gradient is bounded per obs column
    (col_err): a whole-tensor norm dilutes an error confined to one column by about sqrt(O).
 3. The z1 operand image that the l1 kernel writes for the W_ih product (smallk for O <= 32, the wgmma epilogue for
    O >= 64 with T·B >= 32), bit for bit against the bf16 hi / lo split of z1; where no image is due, its region stays
    untouched.
 4. Learner iterations at O from 1 to 1101 against oracle/ref_port.py.
 5. The replay gather (float4 rows when O % 4 == 0, single floats otherwise), local and global per draw, bit for bit.
 6. r2d2_policy_step at O = 1, 4 and 512 (the last 512-wide staged chunk exactly full).

Which kernel served each kernel-level case is observed under torch.profiler in one fresh process (the `routes` fixture,
as in tests/test_gpu_hidden_size.py); the values are checked here.  Run with -s for the routes seen and the worst errors
per group."""
import json
import math
from collections import Counter, defaultdict

import numpy as np
import pytest
import torch

from conftest import rel_l2
from kernel_harness import WorstLog, dev, f64, make_params, num_sms, scan_status, smem_optin
from kernel_harness import nv_routes as nv  # noqa: F401
from learner_harness import col_err, episode
from oracle import actor_oracle
from oracle import learner_oracle as lo
from oracle import ref_port
from oracle.actor_oracle import NETS, policy_params
from oracle.sumtree import SumTreeOracle
from route_check import (ROUTE_KERNELS, RouteLog, launch_counts, observe_in_fresh_process, parse_route, ran,
                         template_args)

pytestmark = pytest.mark.gpu

TOL_FWD, TOL_BWD, TOL_GEMM, TOL_LEARNER = 2e-5, 5e-5, 2e-5, 1e-3
NT = 0
EPI_TANH = 1
O_BUCKETS = (1, 3, 4, 31, 32, 33, 47, 63, 64, 65, 127, 376, 1101)
SENTINEL = 0x7FC0BEEF            # a NaN bit pattern: what the z1 image region holds before the forward

ROUTES = RouteLog()
WORST = WorstLog()
SEEN = defaultdict(set)          # product -> routes asserted


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    WORST.report()
    for prod, routes in sorted(SEEN.items()):
        print(f"{prod} routes asserted: {sorted(routes)}")
    ROUTES.report()


# ------------------------------------------------------------------------------------------------ expected routes
def split_k(M, N, K):
    """gemm_suggest_split_k in the default mode (gemm.cu:280-292, gemm_tc.cu:295-305)."""
    skinny = K < 64 or N < 32 or M < 32
    tiles = math.ceil(M / 128) * math.ceil(N / (64 if skinny else 128))
    k_tiles = math.ceil(K / 32)
    if tiles >= num_sms() or k_tiles < 16:
        return 1
    s = max(1, min(math.ceil(2 * num_sms() / tiles), k_tiles // 8))
    return min(s, 128 if skinny else 256)


def nt_route(M, N, K):
    """Route of an NT product with one K segment, split_k = 1, 16-byte aligned operands, in the default mode: the thin
    kernels first (gemm_thin.cu:499-530: rowdot4, small-N, small-K), then mma.sync for skinny shapes and wgmma for the
    rest (gemm.cu:320-331)."""
    if N <= 32 and K in (128, 256, 512) and N * K * 4 <= 64 * 1024:
        return "rowdot4"
    NP = 8 if N <= 8 else 16 if N <= 16 else 32
    if N <= 32 and 64 <= K <= 2048 and K % 4 == 0 and NP * math.ceil(K / 128) * 128 * 4 <= smem_optin():
        return "smalln:%d" % NP
    if K <= 32:
        return "smallk"
    return "mma" if (K < 64 or N < 32 or M < 32) else "wgmma"


def tn_route(M, N, K):
    """Route of a TN weight-gradient product C[M, N] += A[K, M]^T B[K, N] at net.cu's split_k: thin_tn_kernel<Q> when
    split-K is on and one side is <= 32 wide (gemm_thin.cu:482-498; the narrow side is M when M <= 32 and either N > 32
    or M <= N), otherwise mma.sync for skinny shapes and wgmma for the rest."""
    if split_k(M, N, K) > 1 and (M <= 32 or N <= 32):
        Q = M if (M <= 32 and (N > 32 or M <= N)) else N
        return "thin_tn:%d" % (8 if Q <= 8 else 16 if Q <= 16 else 24 if Q <= 24 else 32)
    return "mma" if (K < 64 or N < 32 or M < 32) else "wgmma"


def z1_image_written(M, H, O):
    """gemm_emits_operand_image (gemm.cu:273-278) for the actor's l1: the small-K kernel or the wgmma epilogue took it
    and H is a multiple of 32 above 32."""
    return H > 32 and H % 32 == 0 and nt_route(M, H, O) in ("smallk", "wgmma")


# ------------------------------------------------------------------------------------------------ 1. actor l1 GEMM
def l1_launch(nv, M, N, O, obs, W1, b1, C):
    return lambda: nv.check(nv.lib().r2d2_gemm_f32(
        NT, M, N, O, obs.data_ptr(), O, W1.data_ptr(), O, None, 0, None, 0, 0, C.data_ptr(), N, b1.data_ptr(), None, 0,
        EPI_TANH, 1, nv.current_stream()))


L1_CASES = ([(O, M, N) for O in O_BUCKETS for M in (1000, 4099) for N in (64, 256)] +
            [(O, M, 64) for O in (64, 376, 1101) for M in (1, 31)])     # fewer than 32 rows: mma.sync at any O


@pytest.mark.parametrize("O,M,N", L1_CASES)
def test_actor_l1(nv, routes, O, M, N):
    rng = np.random.default_rng(O * 10007 + M * 3 + N)
    obs = rng.standard_normal((M, O)).astype(np.float32)
    W1 = (rng.uniform(-1, 1, (N, O)) / np.sqrt(O)).astype(np.float32)
    b1 = rng.uniform(-0.2, 0.2, N).astype(np.float32)
    ref = np.tanh(f64(obs) @ f64(W1).T + f64(b1))
    case = f"l1 O={O} M={M} N={N}"
    route = nt_route(M, N, O)
    ROUTES.assert_route(case, route, routes[case])
    SEEN["actor l1"].add(route)
    C = torch.full((M, N), float("nan"), device="cuda")
    l1_launch(nv, M, N, O, dev(obs), dev(W1), dev(b1), C)()
    WORST.bound("l1", case, C.cpu().numpy(), ref, TOL_GEMM, tile=128, tile_axis=0)


# ------------------------------------------------------------------------------------------------ 2. chains
class Chain:
    """Device buffers of one r2d2_lstm_net_forward / _backward call (repeat 1, head from row 0).  The z1 image region
    (the workspace's last sub-buffer, ChainWs::carve) starts as SENTINEL words, the rest of the workspace as zeros."""

    def __init__(self, nv, O, A, H, critic, T, B, params=None, obs=None, act=None, h0=None, c0=None, d_out=None):
        self.nv, self.lib = nv, nv.lib()
        self.O, self.A, self.H, self.critic, self.T, self.B = O, A, H, critic, T, B
        self.shape = nv.NetShape(O, A, H, int(critic))
        npar = self.lib.r2d2_net_param_count(nv.byref(self.shape))
        z = lambda *s: torch.zeros(s, device="cuda")  # noqa: E731
        self.params = dev(params) if params is not None else z(npar)
        assert self.params.numel() == npar
        self.obs = dev(obs) if obs is not None else z(T, B, O)
        self.act = (dev(act) if act is not None else z(T, B, A)) if critic else None
        self.h0 = dev(h0) if h0 is not None else z(B, H)
        self.c0 = dev(c0) if c0 is not None else z(B, H)
        self.d_out = dev(d_out) if d_out is not None else z(T, B, A)
        n_ws = self.lib.r2d2_net_workspace_floats(nv.byref(self.shape), T, B, 1)
        self.ws = z(n_ws)
        TB, al = T * B, lambda n: (n + 63) // 64 * 64   # noqa: E731
        self.img_floats = al((TB + 127) // 128 * 128 * H)
        self.img = self.ws[n_ws - self.img_floats:]
        self.img.view(torch.int32).fill_(SENTINEL)
        self.out = torch.full((T, B, A), float("nan"), device="cuda")
        self.grads = z(npar)
        self.d_act = torch.full((T, B, A), float("nan"), device="cuda") if critic else None

    def forward(self):
        nv = self.nv
        nv.check(self.lib.r2d2_lstm_net_forward(nv.byref(self.shape), nv.dptr(self.params), nv.dptr(self.obs),
                                                nv.dptr(self.act), nv.dptr(self.h0), nv.dptr(self.c0), self.T, self.B,
                                                1, 0, nv.dptr(self.out), nv.dptr(self.ws), nv.current_stream()))

    def backward(self):
        nv = self.nv
        nv.check(self.lib.r2d2_lstm_net_backward(nv.byref(self.shape), nv.dptr(self.params), nv.dptr(self.obs),
                                                 nv.dptr(self.act), nv.dptr(self.d_out), self.T, self.B, 1, 0,
                                                 nv.dptr(self.grads), nv.dptr(self.d_act), nv.dptr(self.ws),
                                                 nv.current_stream()))

    def run(self):
        self.forward()
        self.backward()


def chain_thin_tn(O, A, H, critic, M):
    """Expected thin_tn_kernel launches {Q: n} of a backward over M = T·B rows (repeat 1, head from row 0): dW3, dW_hh,
    dW_ih, the obs block of dW1 and, for the critic, its action block (net.cu:127-184)."""
    products = [(A, H, M), (4 * H, H, M), (4 * H, H, M), (H, O, M)] + ([(H, A, M)] if critic else [])
    out = Counter()
    for p in products:
        key, args = parse_route(tn_route(*p))
        if key == "thin_tn":
            out[args[0]] += 1
    return dict(out)


def observed_thin_tn(counts):
    out = Counter()
    for name, n in counts.items():
        for args in template_args(name, ROUTE_KERNELS["thin_tn"]):
            out[args[0]] += n
    return dict(out)


CHAIN_TB = (5, 103)                                # T·B = 515: 17 k tiles of 32 (split-K on), 3 rows past 4 x 128
SHORT_TB = (3, 7)                                  # T·B = 21: fewer rows than a 32-row l1 tile, split-K off
CHAIN_H = (32, 64, 128, 512)
CHAIN_CASES = (
    [(O, 3, H, False) + CHAIN_TB for O in O_BUCKETS for H in CHAIN_H] +
    [(O, 3, CHAIN_H[i % 4], True) + CHAIN_TB for i, O in enumerate(O_BUCKETS)] +
    [(40, 3, 32, c) + CHAIN_TB for c in (False, True)] +              # H = 32 <= O: the narrow side of dW1 is M
    [(32, 2, 32, True) + CHAIN_TB, (1101, 5, 512, True) + CHAIN_TB] +
    [(O, 3, 64, c) + SHORT_TB for O in (1, 33, 64, 376) for c in (False, True)])


def chain_key(O, A, H, critic, T, B):
    return f"chain O={O} A={A} H={H} {'critic' if critic else 'actor'} T={T} B={B}"


def bf16_split(z):
    """common.cuh's split_pack2 per element: hi = the bf16 of x rounded half up on the bit pattern, lo = the same of
    x - hi; both as 16-bit words."""
    bits = np.ascontiguousarray(z, np.float32).view(np.uint32)
    h = (bits + np.uint32(0x8000)) & np.uint32(0xFFFF0000)
    r = (z.astype(np.float32) - h.view(np.float32)).astype(np.float32)
    lo = (r.view(np.uint32) + np.uint32(0x8000)) >> np.uint32(16)
    return (h >> np.uint32(16)).astype(np.uint16), lo.astype(np.uint16)


def decode_k_major(img, rows, K):
    """(hi, lo) [rows, K] 16-bit words of a K-major operand image (gemm_tc.cu:41-46): tile (row / 128, k / 32) of 16 KB
    = hi plane + lo plane, each 512 groups of 8 consecutive k of one row; group id = 32 ((row % 128) / 8) +
    8 ((k % 32) / 8) + row % 8."""
    m_tiles = (rows + 127) // 128
    w = img.view(np.uint16)[:m_tiles * (K // 32) * 8192].reshape(m_tiles, K // 32, 2, 512, 8)
    r = np.arange(rows)[:, None]
    k = np.arange(K)[None, :]
    gid = ((r & 127) >> 3) * 32 + ((k & 31) >> 3) * 8 + (r & 7)
    return w[r >> 7, k >> 5, 0, gid, k & 7], w[r >> 7, k >> 5, 1, gid, k & 7]


@pytest.mark.parametrize("O,A,H,critic,T,B", CHAIN_CASES)
def test_chain(nv, routes, O, A, H, critic, T, B):
    M = T * B
    case = chain_key(O, A, H, critic, T, B)
    names = list(routes[case])
    if not critic:
        l1 = nt_route(M, H, O)
        key, args = parse_route(l1)
        assert ran(names, ROUTE_KERNELS[key], args), f"{case}: l1 not on {l1}: {names}"
        SEEN["chain actor l1"].add(l1)
    dw1 = tn_route(H, O, M)
    SEEN["dW1 obs block"].add(dw1)
    want_thin, got_thin = chain_thin_tn(O, A, H, critic, M), observed_thin_tn(routes[case])
    assert got_thin == want_thin, f"{case}: thin_tn launches {got_thin}, expected {want_thin} (dW1 obs on {dw1})"
    if not dw1.startswith("thin_tn"):
        assert ran(names, ROUTE_KERNELS[dw1]), f"{case}: dW1 obs block not on {dw1}: {names}"

    rng = np.random.default_rng(O * 1009 + H * 17 + A * 3 + M + critic)
    p = {k: f64(v) for k, v in make_params(rng, O, A, H, critic).items()}
    obs, act = rng.standard_normal((T, B, O)), rng.uniform(-1, 1, (T, B, A))
    h0, c0 = 0.3 * rng.standard_normal((B, H)), 0.3 * rng.standard_normal((B, H))
    d_out = rng.standard_normal((T, B, A))
    x = np.concatenate((obs, act), 2) if critic else obs
    sv = lo.net_forward(p, f64(x), f64(h0), f64(c0), critic=critic)
    g_ref, dx_ref, _ = lo.net_backward(p, sv, f64(d_out), critic=critic, want_wgrad=True, want_dx=True)

    flat = np.concatenate([np.asarray(p[k], np.float32).reshape(-1) for k in lo.PARAM_KEYS])
    ch = Chain(nv, O, A, H, critic, T, B, params=flat, obs=obs, act=act, h0=h0, c0=c0, d_out=d_out)
    ch.forward()
    torch.cuda.synchronize()
    z1 = ch.ws[:M * H].view(M, H).cpu().numpy()                 # overwritten in place by the backward
    img = ch.img.cpu().numpy()
    ch.backward()
    torch.cuda.synchronize()
    assert scan_status(nv) == 0, f"{case}: a bounded hand-off wait expired inside a scan kernel"

    WORST.bound("chain z1", f"{case} z1", z1, sv["z1"].reshape(M, H), TOL_FWD)
    WORST.bound("chain out", f"{case} out", ch.out.cpu().numpy(), sv["out"], TOL_FWD)
    if critic:
        WORST.bound("chain d_act", f"{case} d_act", ch.d_act.cpu().numpy(), dx_ref[:, :, O:], TOL_BWD, cols=A)
    g, off = ch.grads.cpu().numpy(), 0
    for k in lo.PARAM_KEYS:
        n = g_ref[k].size
        got, want = g[off:off + n].reshape(g_ref[k].shape), g_ref[k]
        off += n
        if k == "l1.weight":
            WORST.bound("chain dW1 obs block", f"{case} grad l1.weight[:, :O]", got[:, :O], want[:, :O], TOL_BWD,
                        cols=O)
            if critic:
                WORST.bound("chain dW1 act block", f"{case} grad l1.weight[:, O:]", got[:, O:], want[:, O:], TOL_BWD,
                            cols=A)
        else:
            WORST.bound(f"chain grad {k}", f"{case} grad {k}", got, want, TOL_BWD)

    # 3. the z1 operand image (the critic's l1 has two K segments: its image follows the same rule at K = O + A)
    K1 = O + (A if critic else 0)
    if z1_image_written(M, H, K1):
        hi, lo_ = decode_k_major(img, M, H)
        want_hi, want_lo = bf16_split(z1)
        for r in range(M):
            assert np.array_equal(hi[r], want_hi[r]) and np.array_equal(lo_[r], want_lo[r]), (
                f"{case}: z1 image row {r} (hi {np.flatnonzero(hi[r] != want_hi[r])[:8]}, "
                f"lo {np.flatnonzero(lo_[r] != want_lo[r])[:8]}) differs from the split of z1")
        SEEN["z1 image"].add(f"written ({nt_route(M, H, K1)})")
    else:
        untouched = img.view(np.uint32) == np.uint32(SENTINEL)
        assert untouched.all(), f"{case}: z1 image region written ({(~untouched).sum()} words) where no image is due"
        SEEN["z1 image"].add(f"not written ({nt_route(M, H, K1)})")


# ------------------------------------------------------------------------------------------------ 4. learner vs port
LEARNER_CASES = [  # obs, act, hidden, batch
    (1, 1, 32, 8), (32, 2, 32, 8), (40, 3, 64, 8), (63, 1, 128, 16), (64, 6, 128, 16), (1101, 4, 128, 8),
]


def _obs_views(block, O):
    return {"l1.weight[:, :O]": np.asarray(block["l1.weight"])[:, :O]}


@pytest.mark.parametrize("obs,act,hidden,batch", LEARNER_CASES)
def test_learner_against_port(obs, act, hidden, batch):
    from r2d2_b200 import engine
    kw = dict(obs=obs, act=act, hidden=hidden, batch=batch, burn_in=2, learning=4, n_step=2)
    pc = ref_port.PathConfig(**kw)
    torch.set_num_threads(max(1, min(32, torch.get_num_threads())))
    port = ref_port.PortLearner(pc, seed=23)
    eng = engine.LearnerEngine(engine.PathConfig(**kw))
    sd = lambda m: {k: v.detach().numpy() for k, v in m.state_dict().items()}  # noqa: E731
    eng.load_state_dicts(sd(port.actor), sd(port.critic))
    for it in range(2):
        batch_np = ref_port.synthetic_batch(pc, seed=700 + it)
        ref = port.iteration(batch_np)
        eng.set_batch(batch_np)
        eng.step()
        torch.cuda.synchronize()
        errs = {}
        for name, got, want in (("q", eng.q_value, ref["q_value"]),
                                ("target", eng.target_q_value, ref["target_q_value"])):
            got = got.cpu().numpy()
            errs[name] = max(rel_l2(got, want), col_err(got, want, act))
        errs["prio"] = rel_l2(eng.priority.cpu().numpy(), ref["priority"])
        errs["critic_loss"] = abs(eng.losses[0].item() - ref["critic_loss"]) / abs(ref["critic_loss"])
        errs["actor_loss"] = abs(eng.losses[1].item() - ref["actor_loss"]) / abs(ref["actor_loss"])
        for net in ("actor", "critic"):
            for what, ref_key in (("grads", "grad"), ("params", "after")):
                got = {k: v.detach().cpu().numpy() for k, v in eng.views(net, what).items()}
                want = ref[f"{net}_{ref_key}"]
                for k in engine.PARAM_KEYS:
                    errs[f"{net}_{ref_key}/{k}"] = rel_l2(got[k], want[k])
                gv, wv = _obs_views(got, obs), _obs_views(want, obs)
                for k in wv:
                    errs[f"{net}_{ref_key}/{k} per column"] = col_err(gv[k], wv[k], obs)
        WORST.note("learner", *errs.values())
        bad = {k: f"{v:.2e}" for k, v in errs.items() if not v < TOL_LEARNER}
        assert not bad, f"iteration {it}: {bad}"
    eng.close()


# ------------------------------------------------------------------------------------------------ 5. replay gather
def assert_window(got, ep, s, rows, what):
    """Slot column `got` (obs, act, rew, term [rows, ...] and states [4, 2, H]) against episode `ep` from row s."""
    obs, act, rew, term, states = got
    assert np.array_equal(obs, ep[0][s:s + rows]), f"{what}: obs window"
    assert np.array_equal(act, ep[1][s:s + rows]), f"{what}: act window"
    assert np.array_equal(rew.reshape(-1), ep[2][s:s + rows]), f"{what}: rew window"
    assert np.array_equal(term.reshape(-1), ep[3][s:s + rows]), f"{what}: term window"
    assert np.array_equal(states, ep[4][s]), f"{what}: stored state"


@pytest.mark.parametrize("O", [1, 3, 4, 64, 1101])
def test_replay_gather_obs_rows(O):
    """O % 4 == 0 moves the obs rows as float4, O = 1, 3 and 1101 one float at a time (act = 3: single floats too)."""
    from r2d2_b200 import engine as E
    cfg = E.PathConfig(obs=O, act=3, hidden=32, batch=64, burn_in=6, learning=10, n_step=3)
    rng = np.random.default_rng(O)
    cap = 12000
    rp = E.DeviceReplay(cfg, capacity_rows=cap)
    oracle = SumTreeOracle(cap)
    eps, row = [], 0
    for n in rng.integers(20, 200, size=50):
        ep = episode(rng, cfg, int(n), zero_pad=True)
        rp.add_episode(*ep)
        oracle.set_range(row, ep[5])
        oracle.set_range(row + len(ep[5]), None, ep[0].shape[0] - len(ep[5]))
        eps.append((row, ep))
        row += ep[0].shape[0]
    u = rng.uniform(size=cfg.batch).astype(np.float32)
    eng = E.LearnerEngine(cfg)
    rp.sample_into(eng, u=torch.as_tensor(u).cuda())
    torch.cuda.synchronize()
    li = eng.leaf_idx.cpu().numpy()
    assert np.array_equal(li, oracle.sample(u))
    ep_i, seq_i = rp.decode(li)
    obs, act, rew, term, states = (t.cpu().numpy() for t in (eng.obs, eng.act, eng.rew, eng.term, eng.states))
    for b in range(cfg.batch):
        row0, ep = eps[ep_i[b]]
        assert row0 + seq_i[b] == li[b]
        assert_window((obs[:, b], act[:, b], rew[:, b], term[:, b], states[:, :, b]), ep, seq_i[b], cfg.rows,
                      f"O={O} sequence {b}")
    rp.close()
    eng.close()


@pytest.mark.parametrize("O", [4, 1101])
def test_global_gather_obs_rows(O):
    """One global draw over two shards (tests/global_harness.py; shard 1's ring wrapped and evicted): every owner's
    per-draw gather stores its rows straight into the consumer's slot.  Each slot column is checked against the host
    episode the draw decodes to, not against a device gather, which shares the copy code."""
    from global_harness import GlobalRun
    from oracle import global_sumtree as gs
    from r2d2_b200 import engine as E
    W = 2
    run = GlobalRun(E, W, dict(obs=O, act=3, hidden=32, batch=16, burn_in=4, learning=6, n_step=2))
    try:
        cfg, B = run.cfg, run.cfg.batch
        run.g.sync()
        lv = run.levels()
        gens = [torch.Generator(device="cuda").manual_seed(40 + r) for r in range(W)]
        us = [torch.rand(B, device="cuda", generator=gen) for gen in gens]
        run.g.sync()
        for stage in (0, 1, 2):
            run.g._issue(lambda r, eng, s, st=stage: run.shards[r].global_draw(eng, st, u=us[r]))
        run.g.sync()
        shard = run.slot_cat("shard").cpu().numpy().astype(np.int64)
        leaf = run.slot_cat("leaf_idx").cpu().numpy()
        ref = gs.global_draw(lv, torch.cat(us).cpu().numpy())
        assert np.array_equal(shard, ref[0]) and np.array_equal(leaf, ref[1])
        assert set(shard.tolist()) == {0, 1}, "both shards hold mass and both are drawn from"
        got = [run.slot_cat(k).cpu().numpy() for k in ("obs", "act", "rew", "term", "states")]
        for j in range(W * B):
            k = int(shard[j])
            ep_i, seq_i = run.shards[k].decode(leaf[j:j + 1])
            held = run.shards[k].stats()["n_episodes"]              # the oldest episodes of a wrapped ring are gone
            assert ep_i[0] >= 0, f"draw {j}: leaf {leaf[j]} lies in no stored episode of shard {k}"
            ep = run.episodes[k][len(run.episodes[k]) - held + int(ep_i[0])]
            assert_window((got[0][:, j], got[1][:, j], got[2][:, j], got[3][:, j], got[4][:, :, j]), ep, int(seq_i[0]),
                          cfg.rows, f"O={O} global draw {j} (shard {k})")
        assert run.status() == [0] * W
    finally:
        run.close()


# ------------------------------------------------------------------------------------------------ 6. policy step
# O = 1: a one-wide staged chunk; O = 512: exactly one full 512-wide chunk of the staged l1 input (policy.cu:116-119)
POLICY_CASES = [(O, 3, 64, 17) for O in (1, 4, 512)]


@pytest.mark.parametrize("O,A,H,N", POLICY_CASES)
def test_policy_step_obs(routes, O, A, H, N):
    from r2d2_b200.policy_step import PolicyStepper
    case = f"policy O={O} A={A} H={H} N={N}"
    ROUTES.assert_route(case, "policy", routes[case])
    missing = [p for p in range(1, 6) if not ran(routes[case], ROUTE_KERNELS["policy"], (p,))]
    assert not missing, f"policy phases {missing} did not run: {routes[case]}"
    md = policy_params(O, A, H, seed=O * 100 + N)
    st = PolicyStepper(O, A, H, N, device="cuda", max_episode_steps=64)
    st.load(md)
    P = {n: {k: v.astype(np.float64) for k, v in md[n].items()} for n in NETS}
    rng = np.random.default_rng(O + A + N)
    ref = np.zeros((4, 2, N, H))
    st.reset(range(N))
    for s in range(60):
        lanes = [n for n in range(N) if s > 0 and s % 30 == (7 * n) % 30]   # staggered episode starts
        if lanes:
            st.reset(lanes)
            ref[:, :, lanes] = 0
        obs = rng.standard_normal((N, O)).astype(np.float32)
        mu = st.step(obs)
        mu_ref, ref = actor_oracle.policy_step(P, obs.astype(np.float64), ref)
        got = st.current_states().cpu().numpy()
        WORST.bound("policy mu", f"O={O} mu step {s}", mu, mu_ref, TOL_FWD, cols=A)
        for k, name in enumerate(NETS):
            WORST.bound("policy h", f"O={O} {name}.h step {s}", got[k, 0], ref[k, 0], TOL_FWD)
            WORST.bound("policy c", f"O={O} {name}.c step {s}", got[k, 1], ref[k, 1], TOL_FWD)


# ------------------------------------------------------------------------------------------------ route observation
def policy_launch(O, A, H, N):
    from r2d2_b200.policy_step import PolicyStepper, policy_step
    st = PolicyStepper(O, A, H, N, device="cuda", max_episode_steps=1)
    return lambda: policy_step(st.params, torch.zeros((N, O), device="cuda"), torch.zeros((4, 2, N, H), device="cuda"),
                               torch.empty((4, 2, N, H), device="cuda"), torch.empty((N, A), device="cuda"))


def route_child(out_path):
    """Entry point of the fresh process behind the `routes` fixture: every case's launch (same entry point, shapes and
    pointer alignment; zero inputs, since no route depends on values) once under the profiler."""
    from r2d2_b200 import native
    native.lib().r2d2_set_scan_impl(1)
    z = lambda *shape: torch.zeros(shape, device="cuda")  # noqa: E731
    out = {}
    for O, M, N in L1_CASES:
        case = f"l1 O={O} M={M} N={N}"
        out[case] = launch_counts(case, l1_launch(native, M, N, O, z(M, O), z(N, O), z(N), z(M, N)))
    for c in CHAIN_CASES:
        case = chain_key(*c)
        out[case] = launch_counts(case, Chain(native, *c).run, agree=True)
    for O, A, H, N in POLICY_CASES:
        case = f"policy O={O} A={A} H={H} N={N}"
        out[case] = launch_counts(case, policy_launch(O, A, H, N))
    with open(out_path, "w") as f:
        json.dump(out, f)


@pytest.fixture(scope="module")
def routes(nv):
    """{case: {route kernel: launches}} observed in a fresh Python process (route_child)."""
    return observe_in_fresh_process("test_gpu_obs_width", timeout=1200)

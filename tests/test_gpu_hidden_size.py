"""Hidden sizes on the GPU: every kernel route that is chosen by the hidden size H (and by the batch at a given H),
checked against float64.

 1. The cluster LSTM scans (r2d2_lstm_scan_forward / _backward).  The dispatcher picks NB = 8, 16 or 32 batch rows per
    cluster from B and from how many clusters of each tile the device keeps resident, so the switch points are found
    by bisection on B (T = 1 chains under the profiler, forward and BPTT apart: their shared memory differs) and
    printed.  Every (H, NB) instantiation then runs at the first B of its tile and at a ragged B inside it: repeat 1
    and 2, dh_head from a later step on, with and without an initial state, head_in requested, dG written over the
    gates.  hs, cs, the gates, head_in, dG and dgin are bounded per tensor, per batch tile (tile_err) and per 32-unit
    group (unit_group_err), since a whole-tensor norm dilutes an error confined to one cluster or one CTA.
 2. The per-step scan path at the H the cluster kernels do not cover, through r2d2_lstm_net_forward / _backward, with
    the routes of its recurrent products asserted.
 3. The small-N heads and d_act at K = H up to 2048, on both sides of the opt-in shared-memory limit of the small-N
    kernel, and learners at those H against the CPU port.
 4. r2d2_policy_step at H that change its grids and O that need several staged input chunks.

Which kernel served each case is observed under torch.profiler in one fresh process (the `routes` fixture: in a
long-lived test process the profiler's collection can stop after the sessions of other test files); the values are
checked here.  Run with -s for the switch points, the (H, NB) cells and routes seen, and the worst errors per group."""
import ctypes
import json
import math

import numpy as np
import pytest
import torch

from conftest import rel_l2
from kernel_harness import WorstLog, dev, f64, make_params, scan_status, smem_optin
from kernel_harness import nv_routes as nv  # noqa: F401
from learner_harness import col_err
from oracle import learner_oracle as lo
from oracle import ref_port
from oracle import actor_oracle
from oracle.actor_oracle import NETS, policy_params
from route_check import ROUTE_KERNELS, RouteLog, observe_in_fresh_process, ran, template_args

pytestmark = pytest.mark.gpu

TOL_FWD, TOL_BWD, TOL_GEMM, TOL_LEARNER = 2e-5, 5e-5, 2e-5, 1e-3
NT, NN = 0, 1
EPI_NONE, EPI_TANH, EPI_MUL_DTANH = 0, 1, 2
CLUSTER_H = (32, 64, 128, 256, 512)
DIRS = ("fwd", "bwd")
KERNEL = {"fwd": ROUTE_KERNELS["scan_fwd"], "bwd": ROUTE_KERNELS["scan_bwd"]}
# instantiations of the cluster kernels: 32-row tiles fit next to the W_hh slice below H = 512 only
INSTANCES = [(H, NB) for H in CLUSTER_H for NB in (8, 16, 32) if not (H == 512 and NB == 32)]
B_MAX = 1 << 17          # bisection ceiling: far beyond any tile switch of an H100

ROUTES = RouteLog()      # asserted routes, reported
PROBES = RouteLog()      # bisection probes, in the route process
WORST = WorstLog()
CELLS = {d: set() for d in DIRS}


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    WORST.report()
    for d in DIRS:
        print(f"{d} (H, NB) cells run: {sorted(CELLS[d])}")
        missing = sorted(set(INSTANCES) - CELLS[d])
        print(f"{d} instantiations not run: {missing if missing else 'none'}")
    ROUTES.report()


# ------------------------------------------------------------------------------------------------ 1. cluster scans
class ScanBuffers:
    """Device buffers of one scan chain; outputs start as NaN so that an unwritten element fails every bound."""

    def __init__(self, T, B, H, repeat, fill=float("nan")):
        S = T * repeat
        self.T, self.B, self.H, self.repeat = T, B, H, repeat
        e = lambda *shape: torch.full(shape, fill, device="cuda")  # noqa: E731
        self.gates, self.hs, self.cs, self.head_in = e(S, B, 4 * H), e(S + 1, B, H), e(S + 1, B, H), e(T, B, H)
        self.dgin = self.gates if repeat == 1 else e(T, B, 4 * H)     # dG is written over the gates (as in the learner)
        self.scratch = torch.empty(B * 4 * H + 64, device="cuda")      # used by the per-step path only

    def forward(self, nv, gin, whh, h0, c0, head=True):
        nv.check(nv.lib().r2d2_lstm_scan_forward(
            nv.dptr(gin), nv.dptr(whh), nv.dptr(h0), nv.dptr(c0), nv.dptr(self.gates), nv.dptr(self.hs),
            nv.dptr(self.cs), nv.dptr(self.head_in) if head else None, self.T, self.B, self.H, self.repeat,
            nv.dptr(self.scratch), nv.current_stream()))

    def backward(self, nv, whh, dh_head, head_first_step):
        nv.check(nv.lib().r2d2_lstm_scan_backward(
            nv.dptr(self.gates), nv.dptr(self.hs), nv.dptr(self.cs), nv.dptr(whh), nv.dptr(dh_head), head_first_step,
            nv.dptr(self.gates), nv.dptr(self.dgin), self.T, self.B, self.H, self.repeat, nv.dptr(self.scratch),
            nv.current_stream()))


_NB_CACHE = {}


def probe_nb(nv, direction, H, B):
    """NB of the `direction` cluster kernel that serves a T = 1 chain of B rows at H (profiled)."""
    key = (direction, H, B)
    if key in _NB_CACHE:
        return _NB_CACHE[key]
    buf = ScanBuffers(1, B, H, 1, fill=0.0)
    gin = torch.zeros((1, B, 4 * H), device="cuda")
    whh = torch.zeros((4 * H, H), device="cuda")
    if direction == "bwd":
        buf.forward(nv, gin, whh, None, None, head=False)
        dh = torch.zeros((1, B, H), device="cuda")
        fn = lambda: buf.backward(nv, whh, dh, 0)  # noqa: E731
    else:
        fn = lambda: buf.forward(nv, gin, whh, None, None, head=False)  # noqa: E731
    _, names = PROBES.profile(f"probe {direction} H={H} B={B}", fn)
    args = [a for n in names for a in template_args(n, KERNEL[direction])]
    assert len(args) == 1 and args[0][0] == H, f"{direction} H={H} B={B}: one {KERNEL[direction]}<{H}, NB>, ran {names}"
    _NB_CACHE[key] = args[0][1]
    return args[0][1]


def first_b(nv, direction, H, lo_b, pred):
    """Smallest B > lo_b with pred(NB(B)), pred monotone in B and false at lo_b; None if not reached by B_MAX."""
    hi = max(2 * lo_b, 8)
    while not pred(probe_nb(nv, direction, H, hi)):
        lo_b = hi
        if hi >= B_MAX:
            return None
        hi = min(2 * hi, B_MAX)
    while hi - lo_b > 1:
        mid = (lo_b + hi) // 2
        if pred(probe_nb(nv, direction, H, mid)):
            hi = mid
        else:
            lo_b = mid
    return hi


def find_switch_points(nv):
    """{(direction, H): {NB: first B of the NB tile}}, by bisection on B; an NB that no B up to B_MAX selects is
    absent."""
    out = {}
    for direction in DIRS:
        for H in CLUSTER_H:
            assert probe_nb(nv, direction, H, 1) == 8, f"{direction} H={H}: B = 1 does not run the 8-row tile"
            tiles = {8: 1}
            b16 = first_b(nv, direction, H, 1, lambda nb: nb >= 16)
            if b16 is not None and probe_nb(nv, direction, H, b16) == 16:
                tiles[16] = b16
            if H != 512:
                b32 = first_b(nv, direction, H, b16 - 1 if b16 else 1, lambda nb: nb >= 32)
                if b32 is not None:
                    tiles[32] = b32
            out[(direction, H)] = tiles
    return out


def tile_cases(switch, direction, H, NB):
    """(first B of the NB tile, a ragged B inside it), or None if the device never selects the tile."""
    tiles = switch[(direction, H)]
    if NB not in tiles:
        return None
    first = tiles[NB]
    nxt = min([b for nb, b in tiles.items() if nb > NB], default=None)
    mid = (first + nxt - 1) // 2 if nxt else first + 2 * NB + NB // 2 + 1
    if mid % NB == 0:
        mid = mid - 1 if mid - 1 > first else mid + 1
    return first, mid


# (T, repeat, initial state given, head_first_step): T = 16 cell steps in both
VARIANTS = [(16, 1, True, 3), (8, 2, False, 5)]


def scan_inputs(H, B, T, repeat, state, hfs, seed):
    rng = np.random.default_rng(seed)
    f32 = lambda a: np.asarray(a, np.float32)  # noqa: E731
    gin = f32(0.5 * rng.standard_normal((T, B, 4 * H)))
    whh = f32(rng.uniform(-1, 1, (4 * H, H)) * 2 / np.sqrt(4 * H))
    h0 = f32(0.3 * rng.standard_normal((B, H))) if state else None
    c0 = f32(0.3 * rng.standard_normal((B, H))) if state else None
    dh_head = f32(rng.standard_normal(((T * repeat - hfs) // repeat, B, H)))
    return gin, whh, h0, c0, dh_head


def run_scan_chain(nv, direction, H, B, NB, T, repeat, state, hfs):
    """Forward (head_in requested) then BPTT with dG over the gates, twice; route, bits and float64 bounds."""
    gin, whh, h0, c0, dh_head = scan_inputs(H, B, T, repeat, state, hfs, seed=H * 7919 + B * 3 + repeat)
    d_gin, d_whh, d_h0, d_c0, d_dh = (None if a is None else dev(a) for a in (gin, whh, h0, c0, dh_head))
    runs = []
    for attempt in range(2):
        buf = ScanBuffers(T, B, H, repeat)
        buf.forward(nv, d_gin, d_whh, d_h0, d_c0)
        gates = buf.gates.clone()
        buf.backward(nv, d_whh, d_dh, hfs)
        torch.cuda.synchronize()
        runs.append({"hs": buf.hs, "cs": buf.cs, "gates": gates, "head_in": buf.head_in, "dgates": buf.gates,
                     "dgin": buf.dgin})
        runs[-1] = {k: v.cpu().numpy() for k, v in runs[-1].items()}
    assert scan_status(nv) == 0, "a bounded hand-off wait expired inside a scan kernel"
    for k in runs[0]:
        assert np.array_equal(runs[0][k].view(np.uint32), runs[1][k].view(np.uint32)), f"{k}: two runs differ"
    CELLS[direction].add((H, NB))
    ref = lo.lstm_scan(*(None if a is None else f64(a) for a in (gin, whh, h0, c0, dh_head)), repeat=repeat,
                       head_first_step=hfs)
    got = runs[0]
    for k, tol in (("hs", TOL_FWD), ("cs", TOL_FWD), ("gates", TOL_FWD), ("head_in", TOL_FWD), ("dgates", TOL_BWD),
                   ("dgin", TOL_BWD)):
        WORST.bound(f"scan {k}", f"H={H} B={B} NB={NB} repeat={repeat} {k}", got[k], ref[k], tol, tile=NB, H=H)


SCAN_CASES = [(d, H, NB, where) for d in DIRS for (H, NB) in INSTANCES for where in ("first", "ragged")]


@pytest.mark.parametrize("direction,H,NB,where", SCAN_CASES)
def test_scan_tile(nv, routes, direction, H, NB, where):
    switch = routes["switch"]
    cases = tile_cases(switch, direction, H, NB)
    assert cases is not None, (f"{KERNEL[direction]}<{H}, {NB}> is unreachable on this device: no B up to {B_MAX} "
                               f"selects it (switch points {switch[(direction, H)]})")
    B = cases[0] if where == "first" else cases[1]
    case = f"scan {direction} H={H} B={B}"
    ROUTES.assert_route(case, f"scan_{direction}:{H},{NB}", routes[case])
    for T, repeat, state, hfs in VARIANTS:
        run_scan_chain(nv, direction, H, B, NB, T, repeat, state, hfs)


# ------------------------------------------------------------------------------------------------ 2. per-step path
def per_step_routes(H, B):
    """Routes of the per-step path's recurrent products in the default mode: forward h W_hh^T + gin (NT, N = 4H,
    K = H, add-Z epilogue) and BPTT dG W_hh (NN, N = H, K = 4H), M = B."""
    fwd = "smallk" if H <= 32 else "mma" if (H < 64 or B < 32) else "wgmma"
    if H <= 8:
        bwd = "smallk"
    elif 16 <= H <= 32:
        bwd = "smalln:%d" % (16 if H <= 16 else 32)
    elif H < 32 or B < 32:
        bwd = "mma"
    else:
        bwd = "wgmma"
    return fwd, bwd


def per_step_launches(nv, H, B):
    """{case: launch} of the bare per-step scan, forward and BPTT, T = 2, at (H, B)."""
    T = 2
    gin, whh = torch.zeros((T, B, 4 * H), device="cuda"), torch.zeros((4 * H, H), device="cuda")
    dh = torch.zeros((T, B, H), device="cuda")
    buf = ScanBuffers(T, B, H, 1, fill=0.0)
    return {f"per-step fwd H={H} B={B}": lambda: buf.forward(nv, gin, whh, None, None),
            f"per-step bwd H={H} B={B}": lambda: buf.backward(nv, whh, dh, 0)}


UNIT_AXIS = {"l1.weight": 0, "l1.bias": 0, "l2.weight_ih": 0, "l2.weight_hh": 0, "l2.bias_ih": 0, "l2.bias_hh": 0,
             "l3.weight": 1, "l3.bias": None}
PER_STEP_H = (8, 12, 16, 20, 28, 36, 48, 160, 384, 480)
# O, A, B, T, repeat, critic, first_row
NET_CASES = [(H, O, A, B, T, repeat, critic, first_row) for H in PER_STEP_H for B in (5, 40)
             for (O, A, T, repeat, critic, first_row) in ((7, 3, 6, 1, True, 1), (6, 2, 5, 2, False, 2))]


@pytest.mark.parametrize("H,O,A,B,T,repeat,critic,first_row", NET_CASES)
def test_net_per_step_path(nv, routes, H, O, A, B, T, repeat, critic, first_row):
    for direction, route in zip(DIRS, per_step_routes(H, B)):
        case = f"per-step {direction} H={H} B={B}"
        ROUTES.assert_route(case, route, routes[case], others=(f"cell_{direction}",))
    rng = np.random.default_rng(H * 1000 + B * 10 + critic)
    p = {k: f64(v) for k, v in make_params(rng, O, A, H, critic).items()}
    obs, act = rng.standard_normal((T, B, O)), rng.uniform(-1, 1, (T, B, A))
    h0, c0 = 0.3 * rng.standard_normal((B, H)), 0.3 * rng.standard_normal((B, H))
    x = np.concatenate((obs, act), 2) if critic else obs
    sv = lo.net_forward(p, f64(x), f64(h0), f64(c0), critic=critic, repeat=repeat)
    out_ref = sv["out"][repeat - 1::repeat][first_row:]
    d_out_rows = rng.standard_normal(out_ref.shape)
    d_out_full = np.zeros_like(sv["out"])
    d_out_full[repeat - 1::repeat][first_row:] = f64(d_out_rows)
    g_ref, dx_ref, _ = lo.net_backward(p, sv, d_out_full, critic=critic, want_wgrad=True, want_dx=True)

    shape = nv.NetShape(O, A, H, int(critic))
    lib = nv.lib()
    flat = np.concatenate([np.asarray(p[k], np.float32).reshape(-1) for k in lo.PARAM_KEYS])
    npar = lib.r2d2_net_param_count(nv.byref(shape))
    assert npar == flat.size
    ws = torch.zeros(lib.r2d2_net_workspace_floats(nv.byref(shape), T, B, repeat), device="cuda")
    dparams, dobs, dact, dh0, dc0 = dev(flat), dev(obs), dev(act), dev(h0), dev(c0)
    out = torch.full(((T - first_row), B, A), float("nan"), device="cuda")
    nv.check(lib.r2d2_lstm_net_forward(nv.byref(shape), nv.dptr(dparams), nv.dptr(dobs),
                                       nv.dptr(dact) if critic else None,
                                       nv.dptr(dh0), nv.dptr(dc0), T, B, repeat, first_row, nv.dptr(out), nv.dptr(ws),
                                       nv.current_stream()))
    grads = torch.zeros(npar, device="cuda")
    d_act = torch.full((T, B, A), float("nan"), device="cuda") if critic else None
    d_out_dev = dev(d_out_rows)
    nv.check(lib.r2d2_lstm_net_backward(nv.byref(shape), nv.dptr(dparams), nv.dptr(dobs),
                                        nv.dptr(dact) if critic else None, nv.dptr(d_out_dev), T, B, repeat, first_row,
                                        nv.dptr(grads), nv.dptr(d_act), nv.dptr(ws), nv.current_stream()))
    torch.cuda.synchronize()
    case = f"H={H} B={B} {'critic' if critic else 'actor'}"
    WORST.bound("per-step out", f"{case} out", out.cpu().numpy(), out_ref, TOL_FWD)
    if critic:
        WORST.bound("per-step d_act", f"{case} d_act", d_act.cpu().numpy(), dx_ref[:, :, O:], TOL_BWD)
    g = grads.cpu().numpy()
    off = 0
    for k in lo.PARAM_KEYS:
        n = g_ref[k].size
        ax = UNIT_AXIS[k]
        WORST.bound(f"per-step grad {k}", f"{case} grad {k}", g[off:off + n].reshape(g_ref[k].shape), g_ref[k], TOL_BWD,
              H=H if ax is not None else None, unit_axis=ax if ax is not None else -1)
        off += n


# ------------------------------------------------------------------------------------------------ 3. heads at K = H
def wide_k_route(N, K):
    """thin_smalln_kernel keeps a [NP][ceil(K / 128) 128] fp32 weight tile in shared memory; a product whose tile
    does not fit the opt-in limit goes to the single-launch mma.sync kernel (N < 32) or to wgmma (N = 32)."""
    NP = 8 if N <= 8 else 16 if N <= 16 else 32
    if NP * math.ceil(K / 128) * 128 * 4 <= smem_optin():
        return "smalln:%d" % NP
    return "mma" if N < 32 else "wgmma"


WIDE_K = (388, 480, 1028, 1792, 1796, 1920, 2048)
HEAD_CASES = [(N, K, epi) for N in (8, 16, 17, 32) for K in WIDE_K for epi in (EPI_NONE, EPI_TANH)]
DACT_CASES = [(N, K) for N in (8, 16, 17, 32) for K in WIDE_K]
GEMM_M, DACT_O = 1031, 17


def head_launch(nv, N, K, epi, h, W3, b3, C):
    return lambda: nv.check(nv.lib().r2d2_gemm_f32(
        NT, GEMM_M, N, K, h.data_ptr(), K, W3.data_ptr(), K, None, 0, None, 0, 0, C.data_ptr(), N, b3.data_ptr(), None,
        0, epi, 1, nv.current_stream()))


def d_act_launch(nv, N, K, dp1, W1, mu, C):
    return lambda: nv.check(nv.lib().r2d2_gemm_f32(
        NN, GEMM_M, N, K, dp1.data_ptr(), K, W1.data_ptr() + 4 * DACT_O, DACT_O + N, None, 0, None, 0, 0,
        C.data_ptr(), N, None, mu.data_ptr(), N, EPI_MUL_DTANH, 1, nv.current_stream()))


@pytest.mark.parametrize("N,K,epi", HEAD_CASES)
def test_head_wide_k(nv, routes, N, K, epi):
    """out = h W3^T + b3 (critic) or tanh of it (actor), M ragged."""
    M = GEMM_M
    rng = np.random.default_rng(N * 10007 + K + epi)
    h = rng.uniform(-1, 1, (M, K)).astype(np.float32)
    W3 = (rng.uniform(-1, 1, (N, K)) / np.sqrt(K)).astype(np.float32)
    b3 = rng.uniform(-0.1, 0.1, N).astype(np.float32)
    ref = f64(h) @ f64(W3).T + f64(b3)
    if epi == EPI_TANH:
        ref = np.tanh(ref)
    case = f"head N={N} K={K} epi={epi}"
    ROUTES.assert_route(case, wide_k_route(N, K), routes[case])
    C = torch.full((M, N), float("nan"), device="cuda")
    d_h, d_w3, d_b3 = dev(h), dev(W3), dev(b3)
    head_launch(nv, N, K, epi, d_h, d_w3, d_b3, C)()
    got = C.cpu().numpy()
    WORST.bound("head", f"head N={N} K={K}", got, ref, TOL_GEMM)
    c = col_err(got, ref, N)
    WORST.note("head col_err", c)
    assert c < TOL_GEMM, f"head N={N} K={K}: col_err {c:.3e}"


@pytest.mark.parametrize("N,K", DACT_CASES)
def test_d_act_wide_k(nv, routes, N, K):
    """d_act = (d(pre-l1) W1[:, O:]) * (1 - mu^2): NN with B pointing O = 17 columns into W1 (ldb = O + N)."""
    M, O = GEMM_M, DACT_O
    I = O + N
    rng = np.random.default_rng(N * 7919 + K)
    dp1 = rng.standard_normal((M, K)).astype(np.float32)
    W1 = (rng.uniform(-1, 1, (K, I)) / np.sqrt(I)).astype(np.float32)
    mu = rng.uniform(-0.95, 0.95, (M, N)).astype(np.float32)
    ref = (f64(dp1) @ f64(W1[:, O:])) * (1.0 - f64(mu) ** 2)
    case = f"d_act N={N} K={K}"
    ROUTES.assert_route(case, wide_k_route(N, K), routes[case])
    C = torch.full((M, N), float("nan"), device="cuda")
    d_dp1, d_w1, d_mu = dev(dp1), dev(W1), dev(mu)
    d_act_launch(nv, N, K, d_dp1, d_w1, d_mu, C)()
    got = C.cpu().numpy()
    WORST.bound("d_act", f"d_act N={N} K={K}", got, ref, TOL_GEMM)
    c = col_err(got, ref, N)
    WORST.note("d_act col_err", c)
    assert c < TOL_GEMM, f"d_act N={N} K={K}: col_err {c:.3e}"


# ------------------------------------------------------------------------------------------------ learner vs port
LEARNER_CASES = [  # obs, act, hidden, batch
    (5, 2, 8, 6), (7, 3, 20, 33), (9, 4, 48, 40), (17, 6, 160, 40), (17, 17, 480, 16),
    (17, 17, 1920, 4),    # heads and d_act with N = 17 at K = 1920: past the small-N kernel's shared memory
]


def _action_views(block, O, A):
    out = {"l3.weight": np.asarray(block["l3.weight"]).T, "l3.bias": np.asarray(block["l3.bias"])}
    if np.asarray(block["l1.weight"]).shape[1] == O + A:
        out["l1.weight[:, O:]"] = np.asarray(block["l1.weight"])[:, O:]
    return out


@pytest.mark.parametrize("obs,act,hidden,batch", LEARNER_CASES)
def test_learner_against_port(obs, act, hidden, batch):
    from r2d2_b200 import engine
    kw = dict(obs=obs, act=act, hidden=hidden, batch=batch, burn_in=2, learning=4, n_step=2)
    pc = ref_port.PathConfig(**kw)
    torch.set_num_threads(max(1, min(32, torch.get_num_threads())))
    port = ref_port.PortLearner(pc, seed=19)
    eng = engine.LearnerEngine(engine.PathConfig(**kw))
    sd = lambda m: {k: v.detach().numpy() for k, v in m.state_dict().items()}  # noqa: E731
    eng.load_state_dicts(sd(port.actor), sd(port.critic))
    for it in range(2):
        batch_np = ref_port.synthetic_batch(pc, seed=500 + it)
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
                gv, wv = _action_views(got, obs, act), _action_views(want, obs, act)
                for k in wv:
                    errs[f"{net}_{ref_key}/{k} per column"] = col_err(gv[k], wv[k], act)
        WORST.note("learner", *errs.values())
        bad = {k: f"{v:.2e}" for k, v in errs.items() if not v < TOL_LEARNER}
        assert not bad, f"iteration {it}: {bad}"
    eng.close()


# ------------------------------------------------------------------------------------------------ 4. policy step
# every H with every O; across the three O of an H, each A and each N once (O = 513 / 1100: two / three KC = 512
# chunks of the staged l1 input)
POLICY_H, POLICY_O, POLICY_A, POLICY_N = (96, 160, 384, 480), (11, 513, 1100), (1, 6, 17), (1, 17, 256)
POLICY_CASES = [(H, O, POLICY_A[(i + j) % 3], POLICY_N[(i + 2 * j) % 3])
                for i, H in enumerate(POLICY_H) for j, O in enumerate(POLICY_O)]


@pytest.mark.parametrize("H,O,A,N", POLICY_CASES)
def test_policy_step_hidden(routes, H, O, A, N):
    from r2d2_b200.policy_step import PolicyStepper
    md = policy_params(O, A, H, seed=H * 100 + O + N)
    st = PolicyStepper(O, A, H, N, device="cuda", max_episode_steps=64)
    st.load(md)
    P = {n: {k: v.astype(np.float64) for k, v in md[n].items()} for n in NETS}
    rng = np.random.default_rng(H + O + A + N)
    case = f"policy H={H} O={O} A={A} N={N}"
    ROUTES.assert_route(case, "policy", routes[case])
    missing = [p for p in range(1, 6) if not ran(routes[case], ROUTE_KERNELS["policy"], (p,))]
    assert not missing, f"policy phases {missing} did not run: {routes[case]}"
    ref = np.zeros((4, 2, N, H))
    st.reset(range(N))
    for s in range(100):
        lanes = [n for n in range(N) if s > 0 and s % 50 == (7 * n) % 50]   # staggered episode starts
        if lanes:
            st.reset(lanes)
            ref[:, :, lanes] = 0
        obs = rng.standard_normal((N, O)).astype(np.float32)
        mu = st.step(obs)
        mu_ref, ref = actor_oracle.policy_step(P, obs.astype(np.float64), ref)
        got = st.current_states().cpu().numpy()
        WORST.bound("policy mu", f"mu step {s}", mu, mu_ref, TOL_FWD)
        for k, name in enumerate(NETS):
            WORST.bound("policy h", f"{name}.h step {s}", got[k, 0], ref[k, 0], TOL_FWD)
            WORST.bound("policy c", f"{name}.c step {s}", got[k, 1], ref[k, 1], TOL_FWD)


def test_policy_lanes_bitwise_independent_h160_o1100():
    from r2d2_b200.policy_step import PolicyStepper, policy_step
    O, A, H, N = 1100, 6, 160, 33
    st = PolicyStepper(O, A, H, 1, device="cuda")
    st.load(policy_params(O, A, H, seed=160))
    g = torch.Generator(device="cuda").manual_seed(0)
    obs = torch.randn((N, O), device="cuda", generator=g)
    s_in = 0.5 * torch.randn((4, 2, N, H), device="cuda", generator=g)

    def step(o, s):
        mu, out = torch.empty((o.shape[0], A), device="cuda"), torch.empty_like(s)
        policy_step(st.params, o, s, out, mu)
        return mu, out
    mu, out = step(obs, s_in)
    mu2, out2 = step(obs, s_in)
    assert torch.equal(mu, mu2) and torch.equal(out, out2), "two runs differ"
    for n in range(N):
        m1, o1 = step(obs[n:n + 1].contiguous(), s_in[:, :, n:n + 1].contiguous())
        assert torch.equal(m1[0], mu[n]) and torch.equal(o1[:, :, 0], out[:, :, n]), f"lane {n} depends on N"


@pytest.mark.parametrize("H", [80, 544])
def test_policy_step_rejects_hidden(nv, H):
    """H = 80 is not a multiple of 32, H = 544 is past the 512 maximum."""
    O, A, N = 5, 2, 4
    buf = torch.zeros(1 << 23, device="cuda")
    p = nv.dptr(buf)
    ptrs = (ctypes.c_void_p * 4)(p.value, p.value, p.value, p.value)
    rc = nv.lib().r2d2_policy_step(nv.byref(nv.NetShape(O, A, H, 0)), ptrs, p, p, nv.dptr(buf[1 << 22:]), p, N, p,
                                   nv.current_stream())
    assert rc == -3
    with pytest.raises(nv.NativeError, match="unsupported shape"):
        nv.check(rc)


# ------------------------------------------------------------------------------------------------ route observation
def policy_launch(H, O, A, N):
    from r2d2_b200.policy_step import PolicyStepper, policy_step
    st = PolicyStepper(O, A, H, N, device="cuda", max_episode_steps=1)
    return lambda: policy_step(st.params, torch.zeros((N, O), device="cuda"), torch.zeros((4, 2, N, H), device="cuda"),
                               torch.empty((4, 2, N, H), device="cuda"), torch.empty((N, A), device="cuda"))


def route_child(out_path):
    """Entry point of the fresh process behind the `routes` fixture: the switch points and every case's launch (same
    entry point, shapes and pointer offsets; zero inputs, since no route depends on values) once under the profiler."""
    from r2d2_b200 import native
    native.lib().r2d2_set_scan_impl(1)
    obs = RouteLog()
    switch = find_switch_points(native)
    names = {}
    for d, H, NB, where in SCAN_CASES:
        cases = tile_cases(switch, d, H, NB)
        if cases:
            B = cases[0] if where == "first" else cases[1]
            probe_nb(native, d, H, B)
            names[f"scan {d} H={H} B={B}"] = PROBES.seen[f"probe {d} H={H} B={B}"]
    launches = {}
    for H, B in sorted({(c[0], c[3]) for c in NET_CASES}):
        launches.update(per_step_launches(native, H, B))
    z = lambda *shape: torch.zeros(shape, device="cuda")  # noqa: E731
    for N, K, epi in HEAD_CASES:
        launches[f"head N={N} K={K} epi={epi}"] = head_launch(native, N, K, epi, z(GEMM_M, K), z(N, K), z(N),
                                                              z(GEMM_M, N))
    for N, K in DACT_CASES:
        launches[f"d_act N={N} K={K}"] = d_act_launch(native, N, K, z(GEMM_M, K), z(K, DACT_O + N), z(GEMM_M, N),
                                                      z(GEMM_M, N))
    for H, O, A, N in POLICY_CASES:
        launches[f"policy H={H} O={O} A={A} N={N}"] = policy_launch(H, O, A, N)
    for case, fn in launches.items():
        names[case] = obs.profile(case, fn)[1]
    out = {"switch": [[d, H, {str(nb): b for nb, b in t.items()}] for (d, H), t in switch.items()], "names": names,
           "probes": len(PROBES.seen), "lost": len(PROBES.lost) + len(obs.lost)}
    with open(out_path, "w") as f:
        json.dump(out, f)


@pytest.fixture(scope="module")
def routes(nv):
    """{case: route kernels that ran} and "switch": {(direction, H): {NB: first B}}, observed in a fresh Python process
    (route_child).  Prints the switch points."""
    got = observe_in_fresh_process("test_gpu_hidden_size", timeout=1200)
    routes = dict(got["names"])
    routes["switch"] = {(d, H): {int(nb): b for nb, b in t.items()} for d, H, t in got["switch"]}
    print(f"\nroute process: {got['probes']} bisection probes, {got['lost']} profiler sessions repeated")
    print("scan tile switch points (first B of each tile):")
    for (d, H), tiles in routes["switch"].items():
        print(f"  {d} H={H:3d}: " + ", ".join(f"NB={nb} from B={b}" for nb, b in sorted(tiles.items())))
    return routes

"""Wide action spaces on the GPU: every kernel route that is chosen by the action count A (or by O + A), checked against
float64 references and the CPU port of the reference at A = 8 .. 64 (dm_control's dog has 38 actions, the Adroit hands
24 to 30; the policy step supports up to 64).

 * the TD / priority kernels through the C ABI, on both sides of the 48 KB shared-memory switch, with NULL outputs and
   importance weights;
 * the learner's A-dependent GEMMs through r2d2_gemm_f32 in the default mode, built the way net.cu builds them (layout,
   leading dimensions, pointer offsets into W1, epilogues), on both sides of every thin-kernel bucket;
 * learner iterations against oracle/ref_port.py, one importance-weighted iteration against oracle/learner_oracle.py;
 * the replay gather, the actor-side priorities and r2d2_policy_step at wide A.

A relative L2 norm over a whole tensor dilutes an error confined to one action column by about sqrt(A), so every output
with an action axis is also bounded per column (col_err).  Each kernel-level case runs under torch.profiler (run_routed)
and asserts the kernel that served it, so a dispatch change that moves a case off its route fails by name instead of
silently dropping the coverage.  Run with -s for the routes seen and the worst errors per group."""
import numpy as np
import pytest
import torch

from conftest import rel_l2
from kernel_harness import WorstLog, dev, f64, ptr, td_inputs
from kernel_harness import nv_routes as nv  # noqa: F401
from learner_harness import col_err, episode, oracle_for
from oracle import actor_oracle
from oracle import learner_oracle as lo
from oracle import ref_port
from oracle.actor_oracle import NETS, policy_params
from oracle.sumtree import SumTreeOracle
from route_check import RouteLog

pytestmark = pytest.mark.gpu

GEMM_TOL = 2e-5
LEARNER_TOL = 1e-3
NT, NN, TN = 0, 1, 2
EPI_NONE, EPI_TANH, EPI_MUL_DTANH = 0, 1, 2

WORST = WorstLog()
ROUTES = RouteLog()
run_routed = ROUTES.run_routed


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    WORST.report()
    ROUTES.report()


@pytest.fixture(scope="module")
def eng_mod():
    from r2d2_b200 import engine
    return engine


def gemm(nv, layout, M, N, K, A, lda, B, ldb, C, ldc, *, A2=None, lda2=0, B2=None, ldb2=0, K2=0, bias=None, Z=None,
         ldz=0, epi=EPI_NONE, split=1):
    """r2d2_gemm_f32 on raw addresses (ints, so that B / B2 / C may point into the middle of a weight block)."""
    nv.check(nv.lib().r2d2_gemm_f32(layout, M, N, K, A, lda, B, ldb, A2, lda2, B2, ldb2, K2, C, ldc, bias, Z, ldz, epi,
                                    split, nv.current_stream()))


# ------------------------------------------------------------------------------------------------ 1. TD / priority
def td_call(nv, inputs, L, B, A, Bn, n, want=("y", "dq", "td", "p", "loss"), w=None):
    """r2d2_td_priority (or _weighted when w is given) with the outputs in `want`, NULL for the others; the requested
    outputs start as NaN so that an unwritten element fails every bound."""
    shapes = {"y": (L, B, A), "dq": (L, B, A), "td": (L, B), "p": (B,), "loss": (1,)}
    o = {k: torch.full(s, float("nan"), device="cuda") for k, s in shapes.items() if k in want}
    q, qn, rew, term = (dev(x) for x in inputs)
    lib, P = nv.lib(), lambda k: ptr(o.get(k))                      # noqa: E731
    if w is None:
        nv.check(lib.r2d2_td_priority(ptr(q), ptr(qn), ptr(rew), ptr(term), L, B, A, Bn, n, 0.997, 0.9, P("y"), P("dq"),
                                      P("td"), P("p"), P("loss"), nv.current_stream()))
    else:
        wt = dev(w)
        nv.check(lib.r2d2_td_priority_weighted(ptr(q), ptr(qn), ptr(rew), ptr(term), ptr(wt), L, B, A, Bn, n, 0.997,
                                               0.9, P("y"), P("dq"), P("td"), P("p"), P("loss"), nv.current_stream()))
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in o.items()}


def check_td(group, o, ref, A):
    y, loss, dq, td_sq, prio = ref
    if "y" in o:
        WORST.bound(group, "target", o["y"], y, 1e-6, cols=A)
    if "dq" in o:
        WORST.bound(group, "dq", o["dq"], dq, 1e-5, cols=A)
    if "td" in o:
        WORST.bound(group, "td_sq", o["td"], td_sq, 1e-5)
    if "p" in o:
        WORST.bound(group, "priority", o["p"], prio, 1e-5)
    if "loss" in o:
        assert abs(o["loss"][0] - loss) < 1e-5 * abs(loss), (o["loss"][0], loss)


# A <= 24: td_elem_kernel + td_reduce_kernel (8 warps x 2 x 32 x A floats of shared memory <= 48 KB, A = 24 exactly);
# A > 24: td_priority_column_kernel.  B ragged against the 32-wide column blocks, L ragged against 32 and 8 warps.
TD_CASES = [(A, B, L, n, "td_two_pass" if A <= 24 else "td_column")
            for A in (24, 25, 32, 33, 38, 64) for B in (1, 31, 33, 257) for L in (2, 33, 80) for n in (1, 5)]


@pytest.mark.parametrize("A,B,L,n,route", TD_CASES)
def test_td_priority_wide(nv, A, B, L, n, route):
    Bn = 3
    inputs = td_inputs(L, B, A, Bn, n, seed=A * 10007 + B * 101 + L * 7 + n)
    ref = lo.td_targets_and_priorities(*(f64(x) for x in inputs), burn_in=Bn, learning=L, n_step=n, gamma=0.997)
    o = run_routed(f"td A={A} B={B} L={L} n={n}", route, lambda: td_call(nv, inputs, L, B, A, Bn, n))
    check_td("td", o, ref, A)


# td_sq = NULL forces the column kernel at any A ("any output pointer may be NULL"); each of the other outputs NULL in
# turn keeps the two-pass route.  Every output still requested meets the same bounds.
NULL_CASES = [(("y", "dq", "p", "loss"), "td_column"), (("dq", "td", "p", "loss"), "td_two_pass"),
              (("y", "td", "p", "loss"), "td_two_pass"), (("y", "dq", "td", "loss"), "td_two_pass"),
              (("y", "dq", "td", "p"), "td_two_pass")]


@pytest.mark.parametrize("want,route", NULL_CASES, ids=["no_td_sq", "no_target", "no_dq", "no_priority", "no_loss"])
def test_td_priority_null_outputs(nv, want, route):
    A, B, L, n, Bn = 6, 33, 33, 5, 3
    inputs = td_inputs(L, B, A, Bn, n, seed=5)
    ref = lo.td_targets_and_priorities(*(f64(x) for x in inputs), burn_in=Bn, learning=L, n_step=n, gamma=0.997)
    o = run_routed(f"td A=6 only {','.join(want)}", route, lambda: td_call(nv, inputs, L, B, A, Bn, n, want=want))
    assert set(o) == set(want)
    check_td("td_null_outputs", o, ref, A)


@pytest.mark.parametrize("A", [25, 64])
def test_td_priority_weighted_wide(nv, A):
    """The column kernel's is_weight branch: dq and the loss weighted per sequence, td_sq and the priorities the bits
    of the unweighted call on the same route."""
    B, L, n, Bn = 33, 33, 5, 3
    inputs = td_inputs(L, B, A, Bn, n, seed=A)
    w = np.random.default_rng(A + 1).uniform(0.05, 1.0, B).astype(np.float32)
    ref = lo.td_targets_and_priorities(*(f64(x) for x in inputs), burn_in=Bn, learning=L, n_step=n, gamma=0.997,
                                       is_weight=f64(w))
    o = run_routed(f"td weighted A={A}", "td_column", lambda: td_call(nv, inputs, L, B, A, Bn, n, w=w))
    check_td("td_weighted", o, ref, A)
    plain = td_call(nv, inputs, L, B, A, Bn, n)
    assert np.array_equal(o["td"].view(np.uint32), plain["td"].view(np.uint32))
    assert np.array_equal(o["p"].view(np.uint32), plain["p"].view(np.uint32))


# ------------------------------------------------------------------------------------------------ 2. GEMMs
# critic l1: z1 = tanh(obs W1[:, :O]^T + act W1[:, O:]^T + b1), two K segments, B2 = W1 + O, ldb = ldb2 = O + A.
# O + A <= 32: small-K streaming kernel; 33 .. 63: mma.sync (skinny K); >= 64: wgmma with two packs per operand.
L1_CASES = [(O, A, N, route) for (O, A, route) in ((7, 25, "smallk"), (8, 25, "mma"), (25, 38, "mma"), (26, 38, "wgmma"))
            for N in (64, 96, 256)]


@pytest.mark.parametrize("O,A,N,route", L1_CASES)
def test_critic_l1_two_segments(nv, O, A, N, route):
    M, I = 4097, O + A
    rng = np.random.default_rng(O * 1000 + A * 10 + N)
    obs, act = rng.standard_normal((M, O)).astype(np.float32), rng.uniform(-1, 1, (M, A)).astype(np.float32)
    W1 = rng.uniform(-1, 1, (N, I)).astype(np.float32) / np.sqrt(I)
    b1 = rng.uniform(-0.2, 0.2, N).astype(np.float32)
    ref = np.tanh(f64(obs) @ f64(W1[:, :O]).T + f64(act) @ f64(W1[:, O:]).T + b1)
    d_obs, d_act, d_w1, d_b1 = dev(obs), dev(act), dev(W1), dev(b1)
    C = torch.full((M, N), float("nan"), device="cuda")
    run_routed(f"critic l1 O={O} A={A} N={N}", route, lambda: gemm(
        nv, NT, M, N, O, ptr(d_obs), O, ptr(d_w1), I, ptr(C), N, A2=ptr(d_act), lda2=A, B2=ptr(d_w1, O), ldb2=I, K2=A,
        bias=ptr(d_b1), epi=EPI_TANH))
    WORST.bound("critic_l1", "z1", C.cpu().numpy(), ref, GEMM_TOL)


HEAD_A = (8, 9, 16, 17, 24, 25, 32, 33, 64)


def thin_n_route(A, K):
    """Route of an NT / NN product with N = A outputs per row and reduction K = H (heads, d_act), default mode."""
    if A > 32:
        return "wgmma"
    if K in (128, 256, 512) and A * K * 4 <= 64 * 1024:
        return "rowdot4"
    return "smalln:%d" % (8 if A <= 8 else 16 if A <= 16 else 32)


# heads: out = h W3^T + b3 (critic) or tanh of it (actor), M = T*B rows with a ragged tail
HEAD_CASES = [(A, H, epi, thin_n_route(A, H)) for A in HEAD_A for H in (64, 96, 128, 512) for epi in (EPI_NONE, EPI_TANH)]


@pytest.mark.parametrize("A,H,epi,route", HEAD_CASES)
def test_head_forward(nv, A, H, epi, route):
    M = 4099
    rng = np.random.default_rng(A * 1000 + H + epi)
    h = rng.uniform(-1, 1, (M, H)).astype(np.float32)
    W3 = rng.uniform(-1, 1, (A, H)).astype(np.float32) / np.sqrt(H)
    b3 = rng.uniform(-0.1, 0.1, A).astype(np.float32)
    ref = f64(h) @ f64(W3).T + b3
    if epi == EPI_TANH:
        ref = np.tanh(ref)
    d_h, d_w3, d_b3 = dev(h), dev(W3), dev(b3)
    C = torch.full((M, A), float("nan"), device="cuda")
    run_routed(f"head A={A} H={H} epi={epi}", route, lambda: gemm(
        nv, NT, M, A, H, ptr(d_h), H, ptr(d_w3), H, ptr(C), A, bias=ptr(d_b3), epi=epi))
    WORST.bound("head", "out", C.cpu().numpy(), ref, GEMM_TOL, cols=A)


# d_act = (d(pre-l1) W1[:, O:]) * (1 - mu^2): NN with B = W1 + O, ldb = O + A; O = 17 / 20 / 24 puts B 68 / 80 / 96 bytes
# past the weight block (4-, 16- and 32-byte aligned)
DACT_CASES = [(O, A, H, thin_n_route(A, H)) for O in (17, 20, 24) for A in HEAD_A for H in (96, 256)]


@pytest.mark.parametrize("O,A,H,route", DACT_CASES)
def test_d_act(nv, O, A, H, route):
    M, I = 4099, O + A
    rng = np.random.default_rng(O * 997 + A * 31 + H)
    dp1 = rng.standard_normal((M, H)).astype(np.float32)
    W1 = rng.uniform(-1, 1, (H, I)).astype(np.float32) / np.sqrt(I)
    mu = rng.uniform(-0.95, 0.95, (M, A)).astype(np.float32)
    ref = (f64(dp1) @ f64(W1[:, O:])) * (1.0 - f64(mu) ** 2)
    d_dp1, d_w1, d_mu = dev(dp1), dev(W1), dev(mu)
    C = torch.full((M, A), float("nan"), device="cuda")
    run_routed(f"d_act O={O} A={A} H={H}", route, lambda: gemm(
        nv, NN, M, A, H, ptr(d_dp1), H, ptr(d_w1, O), I, ptr(C), A, Z=ptr(d_mu), ldz=A, epi=EPI_MUL_DTANH))
    WORST.bound("d_act", "d_act", C.cpu().numpy(), ref, GEMM_TOL, cols=A)


def tn_route(A):
    return "wgmma" if A > 32 else "thin_tn:%d" % (8 if A <= 8 else 16 if A <= 16 else 24 if A <= 24 else 32)


# dW3 (TN, M = A, N = H) and the dW1 action block (TN, M = H, N = A, C = dW1 + O with ldc = O + A), split-K adding into
# C as the learner's zeroed gradient block (here: into random contents, which must survive)
TN_CASES = [(which, A, K, tn_route(A)) for which in ("dW3", "dW1_act") for A in HEAD_A for K in (320, 1920, 20480)]


@pytest.mark.parametrize("which,A,K,route", TN_CASES)
def test_weight_gradient_blocks(nv, which, A, K, route):
    H, O = 256, 17
    split = max(2, min(80, K // 256))
    rng = np.random.default_rng(A * 7919 + K + (which == "dW3"))
    if which == "dW3":
        d_pre = rng.standard_normal((K, A)).astype(np.float32)
        hin = rng.uniform(-1, 1, (K, H)).astype(np.float32)
        ref = f64(d_pre).T @ f64(hin)                                 # [A, H]
        C0 = (rng.standard_normal((A, H)) * ref.std()).astype(np.float32)
        a_op, b_op, C0_dev = dev(d_pre), dev(hin), dev(C0)
        C = torch.empty_like(C0_dev)

        def run():
            C.copy_(C0_dev)
            gemm(nv, TN, A, H, K, ptr(a_op), A, ptr(b_op), H, ptr(C), H, split=split)
        run_routed(f"dW3 A={A} K={K}", route, run)
        got = C.cpu().numpy().astype(np.float64) - C0
        WORST.bound("dW3", "dW3", got.T, ref.T, GEMM_TOL, cols=A)          # per action row
    else:
        z1 = rng.standard_normal((K, H)).astype(np.float32)
        act = rng.uniform(-1, 1, (K, A)).astype(np.float32)
        ref = f64(z1).T @ f64(act)                                    # [H, A]
        C0 = (rng.standard_normal((H, O + A)) * ref.std()).astype(np.float32)
        a_op, b_op, C0_dev = dev(z1), dev(act), dev(C0)
        C = torch.empty_like(C0_dev)

        def run():
            C.copy_(C0_dev)
            gemm(nv, TN, H, A, K, ptr(a_op), H, ptr(b_op), A, ptr(C, O), O + A, split=split)
        run_routed(f"dW1 action block A={A} K={K}", route, run)
        out = C.cpu().numpy()
        assert np.array_equal(out[:, :O], C0[:, :O]), "the obs columns of dW1 were written"
        WORST.bound("dW1_act", "dW1[:, O:]", out[:, O:].astype(np.float64) - C0[:, O:], ref, GEMM_TOL, cols=A)


# ------------------------------------------------------------------------------------------------ 3. learner vs port
def flat_sd(views):
    return {k: v.detach().cpu().numpy() for k, v in views.items()}


def action_views(block, O, A):
    """[-1, A] views of the action-indexed parts of a parameter / gradient dict: l3.weight rows, l3.bias and, for the
    critic, the action columns of l1.weight."""
    out = {"l3.weight": np.asarray(block["l3.weight"]).T, "l3.bias": np.asarray(block["l3.bias"])}
    if np.asarray(block["l1.weight"]).shape[1] == O + A:
        out["l1.weight[:, O:]"] = np.asarray(block["l1.weight"])[:, O:]
    return out


def check_learner(group, eng, eng_mod, ref, O, A):
    errs = {}
    for name, got, want in (("q", eng.q_value, ref["q_value"]), ("target", eng.target_q_value, ref["target_q_value"])):
        got = got.cpu().numpy()
        errs[name] = (rel_l2(got, want), col_err(got, want, A))
    errs["prio"] = (rel_l2(eng.priority.cpu().numpy(), ref["priority"]), 0.0)
    errs["critic_loss"] = (abs(eng.losses[0].item() - ref["critic_loss"]) / abs(ref["critic_loss"]), 0.0)
    errs["actor_loss"] = (abs(eng.losses[1].item() - ref["actor_loss"]) / abs(ref["actor_loss"]), 0.0)
    for net in ("actor", "critic"):
        for what, ref_key in (("grads", "grad"), ("params", "after")):
            got = flat_sd(eng.views(net, what))
            want = ref[f"{net}_{ref_key}"]
            for k in eng_mod.PARAM_KEYS:
                errs[f"{net}_{ref_key}/{k}"] = (rel_l2(got[k], want[k]), 0.0)
            gv, wv = action_views(got, O, A), action_views(want, O, A)
            for k in wv:
                errs[f"{net}_{ref_key}/{k} per column"] = (0.0, col_err(gv[k], wv[k], A))
    WORST.note(f"{group} rel_l2", *(r for r, _ in errs.values()))
    WORST.note(f"{group} col_err", *(c for _, c in errs.values()))
    return {k: v for k, v in errs.items() if not (v[0] < LEARNER_TOL and v[1] < LEARNER_TOL)}


LEARNER_CASES = [
    # obs, act, hidden, batch, burn_in, learning, n_step
    (8, 24, 96, 33, 4, 8, 3),       # largest A on the two-pass TD route, O + A = 32, H on the generic scan path
    (7, 25, 64, 40, 4, 8, 3),       # column TD kernel, small-K critic l1 with K2 = 25, small-N heads
    (24, 38, 128, 64, 8, 16, 3),    # dog-sized: critic l1 on mma.sync (O + A = 62), wgmma heads, d_act with ldb = 62
    (17, 12, 512, 24, 40, 80, 5),   # rowdot4 heads at H = 512, thin_tn with Q = 12 for dW3
    (67, 64, 256, 32, 8, 16, 3),    # the policy maximum A = 64: wgmma with two K segments
]


@pytest.mark.parametrize("obs,act,hidden,batch,burn_in,learning,n_step", LEARNER_CASES)
def test_learner_against_port_wide(eng_mod, obs, act, hidden, batch, burn_in, learning, n_step):
    kw = dict(obs=obs, act=act, hidden=hidden, batch=batch, burn_in=burn_in, learning=learning, n_step=n_step)
    pc = ref_port.PathConfig(**kw)
    torch.set_num_threads(max(1, min(32, torch.get_num_threads())))
    port = ref_port.PortLearner(pc, seed=13)
    eng = eng_mod.LearnerEngine(eng_mod.PathConfig(**kw))
    sd = lambda m: {k: v.detach().numpy() for k, v in m.state_dict().items()}  # noqa: E731
    eng.load_state_dicts(sd(port.actor), sd(port.critic))
    for it in range(2):
        batch_np = ref_port.synthetic_batch(pc, seed=300 + it)
        ref = port.iteration(batch_np)
        eng.set_batch(batch_np)
        eng.step()
        torch.cuda.synchronize()
        bad = check_learner("learner", eng, eng_mod, ref, obs, act)
        assert not bad, f"iteration {it}: {bad}"
    eng.close()


def test_weighted_learner_iteration_column_kernel(eng_mod):
    """One importance-weighted iteration at A = 25 (the column TD kernel's is_weight branch) against the float64 oracle;
    td_sq and the priorities are the bits of the unweighted engine."""
    kw = dict(obs=7, act=25, hidden=64, batch=40, burn_in=4, learning=8, n_step=3)
    pc = ref_port.PathConfig(**kw)
    port = ref_port.PortLearner(pc, seed=17)
    sd = lambda m: {k: v.detach().numpy() for k, v in m.state_dict().items()}  # noqa: E731
    actor, critic = sd(port.actor), sd(port.critic)
    batch = ref_port.synthetic_batch(pc, seed=7)
    w = np.random.default_rng(29).uniform(0.05, 1.0, kw["batch"]).astype(np.float32)
    cfg = eng_mod.PathConfig(**kw, is_exponent=0.6)
    eng = eng_mod.LearnerEngine(cfg)
    eng.load_state_dicts(actor, critic)
    eng.set_batch(dict(batch, is_weight=w))
    eng.step()
    plain = eng_mod.LearnerEngine(eng_mod.PathConfig(**kw))
    plain.load_state_dicts(actor, critic)
    plain.set_batch(batch)
    plain.step()
    torch.cuda.synchronize()
    assert torch.equal(eng.td_sq, plain.td_sq) and torch.equal(eng.priority, plain.priority)
    ref = oracle_for(cfg, actor, critic).iteration(dict(batch, is_weight=w))
    bad = check_learner("learner_weighted", eng, eng_mod, ref, kw["obs"], kw["act"])
    assert not bad, bad
    eng.close()
    plain.close()


# ------------------------------------------------------------------------------------------------ 4. replay / actor side
@pytest.mark.parametrize("A", [25, 32, 64])
def test_replay_gather_wide_action_rows(eng_mod, A):
    """A % 4 == 0 moves the action rows as float4, A = 25 element by element: both bit-exact."""
    cfg = eng_mod.PathConfig(obs=6, act=A, hidden=32, batch=64, burn_in=6, learning=10, n_step=3)
    rng = np.random.default_rng(A)
    cap = 20000
    rp = eng_mod.DeviceReplay(cfg, capacity_rows=cap)
    oracle = SumTreeOracle(cap)
    eps, row = [], 0
    for E in rng.integers(20, 200, size=60):
        ep = episode(rng, cfg, int(E), zero_pad=True)
        rp.add_episode(*ep)
        oracle.set_range(row, ep[5])
        oracle.set_range(row + len(ep[5]), None, ep[0].shape[0] - len(ep[5]))
        eps.append((row, ep))
        row += ep[0].shape[0]
    u = rng.uniform(size=cfg.batch).astype(np.float32)
    eng = eng_mod.LearnerEngine(cfg)
    rp.sample_into(eng, u=torch.as_tensor(u).cuda())
    torch.cuda.synchronize()
    li = eng.leaf_idx.cpu().numpy()
    assert np.array_equal(li, oracle.sample(u))
    ep_i, seq_i = rp.decode(li)
    obs, act, rew, term, states = (t.cpu().numpy() for t in (eng.obs, eng.act, eng.rew, eng.term, eng.states))
    for b in range(cfg.batch):
        row0, ep = eps[ep_i[b]]
        s = seq_i[b]
        assert row0 + s == li[b]
        assert np.array_equal(act[:, b], ep[1][s:s + cfg.rows]), f"act window of sequence {b}"
        assert np.array_equal(obs[:, b], ep[0][s:s + cfg.rows])
        assert np.array_equal(rew[:, b].reshape(-1), ep[2][s:s + cfg.rows])
        assert np.array_equal(term[:, b].reshape(-1), ep[3][s:s + cfg.rows])
        assert np.array_equal(states[:, :, b], ep[4][s])
    rp.close()
    eng.close()


def test_actor_priorities_38_actions():
    """Actor-side n-step sums and initial priorities at A = 38, episodes of different lengths in one batch."""
    from r2d2_b200 import actor_priority as ap
    O, A, H, Bn, L, n, gamma = 24, 38, 64, 20, 40, 5, 0.997
    nets = policy_params(O, A, H, seed=38)
    rng = np.random.default_rng(38)
    episodes = []
    for E in (60, 61, 77, 103, 150):
        obs = rng.standard_normal((E + n, O)).astype(np.float32)
        act = rng.uniform(-1, 1, (E + n, A)).astype(np.float32)
        raw = rng.standard_normal(E + n).astype(np.float32)
        term = np.zeros(E + n, np.float32)
        obs[E:], act[E:], raw[E:], term[E:] = 0, 0, 0, 1
        episodes.append((obs, act, raw, term))
    prios, rews = ap.episode_priorities(nets["critic"], nets["target_actor"], nets["target_critic"], episodes, hidden=H,
                                        burn_in=Bn, learning=L, n_step=n, gamma=gamma, rewards_are_raw=True)
    for (obs, act, raw, term), p, r in zip(episodes, prios, rews):
        want_r = actor_oracle.nstep_rewards(raw, n, gamma)
        assert rel_l2(r, want_r) < 1e-6
        want_p = actor_oracle.episode_priorities(nets["critic"], nets["target_actor"], nets["target_critic"], obs, act,
                                                 want_r, term, burn_in=Bn, learning=L, n_step=n, gamma=gamma)
        assert p.shape == want_p.shape
        if p.size:
            assert rel_l2(p, want_p) < 1e-3, rel_l2(p, want_p)


# N = 17 leaves a 16-lane tile with a single lane; A = 64 is the documented maximum
POLICY_CASES = [(A, N, H) for A in (25, 33, 64) for N in (1, 17, 256) for H in (64, 256)]


@pytest.mark.parametrize("A,N,H", POLICY_CASES)
def test_policy_step_wide(A, N, H):
    from r2d2_b200.policy_step import PolicyStepper
    O = 11
    md = policy_params(O, A, H, seed=A * 100 + N + H)
    st = PolicyStepper(O, A, H, N, device="cuda", max_episode_steps=64)
    st.load(md)
    P = {n: {k: v.astype(np.float64) for k, v in md[n].items()} for n in NETS}
    rng = np.random.default_rng(N + A)
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
        WORST.bound("policy", f"mu step {s}", mu, mu_ref, 2e-5, cols=A)
        for k, name in enumerate(NETS):
            WORST.bound("policy", f"{name}.h step {s}", got[k, 0], ref[k, 0], 2e-5)
            WORST.bound("policy", f"{name}.c step {s}", got[k, 1], ref[k, 1], 2e-5)


def test_policy_lanes_bitwise_independent_64_actions():
    from r2d2_b200.policy_step import PolicyStepper, policy_step
    O, A, H, N = 11, 64, 128, 33
    st = PolicyStepper(O, A, H, 1, device="cuda")
    st.load(policy_params(O, A, H, seed=64))
    g = torch.Generator(device="cuda").manual_seed(0)
    obs = torch.randn((N, O), device="cuda", generator=g)
    s_in = 0.5 * torch.randn((4, 2, N, H), device="cuda", generator=g)

    def step(o, s):
        mu, out = torch.empty((o.shape[0], A), device="cuda"), torch.empty_like(s)
        policy_step(st.params, o, s, out, mu)
        return mu, out
    mu, out = step(obs, s_in)
    for n in range(N):
        m1, o1 = step(obs[n:n + 1].contiguous(), s_in[:, :, n:n + 1].contiguous())
        assert torch.equal(m1[0], mu[n]) and torch.equal(o1[:, :, 0], out[:, :, n]), f"lane {n} depends on N"

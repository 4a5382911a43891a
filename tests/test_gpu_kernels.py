"""GPU parity of the individual kernels, called through the C ABI (ctypes), against float64 numpy
oracles (oracle/learner_oracle.py).  Tolerances are relative L2 per tensor; the path's bar is 1e-3
(BASELINE.json north_star), the kernels are expected to sit near 1e-5 (bf16x3 split, fp32 accumulate)."""
import numpy as np
import pytest
import torch

from conftest import rel_l2
from kernel_harness import dev, nv, scan_status  # noqa: F401
from oracle import learner_oracle as lo

pytestmark = pytest.mark.gpu

TOL = 2e-5


# ----------------------------------------------------------------------------------------------
GEMM_CASES = [
    # layout, M, N, K, K2, bias, epi, split_k
    (0, 128, 64, 32, 0, False, 0, 1),
    (0, 300, 200, 100, 0, True, 1, 1),
    (0, 1000, 256, 17, 6, True, 1, 1),       # critic l1: cat(obs, act) as two K segments, unaligned lda
    (0, 517, 6, 256, 0, True, 0, 1),         # head: tiny N
    (0, 64, 1024, 256, 0, True, 0, 1),
    (1, 300, 200, 100, 0, False, 0, 1),
    (1, 777, 256, 1024, 0, False, 2, 1),     # dgrad with dtanh epilogue
    (1, 513, 130, 6, 0, False, 2, 1),        # K tiny (head dgrad)
    (1, 400, 6, 256, 0, False, 0, 1),        # N tiny (d_act)
    (2, 200, 300, 1000, 0, False, 0, 1),
    (2, 1024, 256, 5000, 0, False, 0, 8),    # wgrad split-K
    (2, 6, 256, 3000, 0, False, 0, 4),       # dW3
    (2, 256, 17, 4000, 0, False, 0, 5),      # dW1 obs block (ldb = 17)
    (0, 100, 64, 40, 0, False, 3, 1),        # add-Z epilogue (generic scan path)
    (0, 4000, 1024, 256, 0, True, 0, 1),     # x*W_ih^T shape (many k tiles, full N tiles)
    (1, 3000, 256, 1024, 0, False, 2, 1),
    (2, 1024, 256, 30720, 0, False, 0, 16),  # dW_hh at cfg-2 size
    (0, 130, 257, 77, 0, True, 1, 1),        # ragged everything
    (1, 257, 130, 77, 0, False, 0, 1),
    (2, 130, 257, 777, 0, False, 0, 3),
    (0, 20480, 256, 17, 0, True, 1, 1),      # actor l1 at cfg-2 size (thin small-K kernel in default mode)
    (0, 4099, 300, 3, 1, True, 1, 1),        # Pendulum critic l1: K = 3 + 1, N not a multiple of 256
    (0, 20481, 6, 256, 0, True, 1, 1),       # actor head at cfg-2 size, odd row count
    (1, 4097, 17, 512, 0, False, 2, 1),      # small-N NN with dtanh epilogue, N = 17
    (0, 999, 1, 128, 0, True, 0, 1),         # Pendulum head, N = 1
    (2, 6, 256, 20480, 0, False, 0, 74),     # dW3 at cfg-2 size
    (2, 256, 17, 32000, 0, False, 0, 120),   # dW1 obs block at cfg-2 size
    (2, 300, 6, 5000, 0, False, 0, 7),       # dW1 action block, wide side not a multiple of 256
]


@pytest.fixture(params=["tc", "mma", "default"])
def gemm_impl(request, nv):
    # 2: wgmma path for every shape; 0: mma.sync kernel; 1 (default): wgmma + the fp32 streaming kernels of
    # gemm_thin.cu for shapes with a dimension <= 32
    nv.lib().r2d2_set_gemm_impl({"tc": 2, "mma": 0, "default": 1}[request.param])
    yield request.param
    nv.lib().r2d2_set_gemm_impl(1)


@pytest.mark.parametrize("layout,M,N,K,K2,bias,epi,split", GEMM_CASES)
def test_gemm(nv, gemm_impl, layout, M, N, K, K2, bias, epi, split):
    rng = np.random.default_rng(hash((layout, M, N, K)) % 2 ** 31)
    if layout == 0:
        A, Bm = rng.standard_normal((M, K)), rng.standard_normal((N, K + K2))
        A2 = rng.standard_normal((M, K2)) if K2 else None
        ref = A @ Bm[:, :K].T + (A2 @ Bm[:, K:].T if K2 else 0)
        lda, ldb = K, K + K2
    elif layout == 1:
        A, Bm = rng.standard_normal((M, K)), rng.standard_normal((K, N))
        A2, ref, lda, ldb = None, A @ Bm, K, N
    else:
        A, Bm = rng.standard_normal((K, M)), rng.standard_normal((K, N))
        A2, ref, lda, ldb = None, A.T @ Bm, M, N
    A, Bm = A.astype(np.float32), Bm.astype(np.float32)
    ref = (A.astype(np.float64) @ Bm[:, :K].astype(np.float64).T if layout == 0 else
           (A.astype(np.float64) @ Bm if layout == 1 else A.astype(np.float64).T @ Bm))
    if K2:
        A2 = A2.astype(np.float32)
        ref = ref + A2.astype(np.float64) @ Bm[:, K:].astype(np.float64).T
    bv = rng.standard_normal(N).astype(np.float32) if bias else None
    Z = (rng.uniform(-0.9, 0.9, (M, N))).astype(np.float32) if epi in (2, 3) else None
    if bias:
        ref = ref + bv
    if epi == 1:
        ref = np.tanh(ref)
    elif epi == 2:
        ref = ref * (1 - Z.astype(np.float64) ** 2)
    elif epi == 3:
        ref = ref + Z
    dA, dB = dev(A), dev(Bm)
    dA2 = dev(A2) if K2 else None
    dC = torch.zeros((M, N), device="cuda")
    dbias = dev(bv) if bias else None
    dZ = dev(Z) if Z is not None else None
    B2ptr = (dB.data_ptr() + 4 * K) if K2 else None
    nv.check(nv.lib().r2d2_gemm_f32(layout, M, N, K, nv.dptr(dA), lda, nv.dptr(dB), ldb,
                                    nv.dptr(dA2), K2, B2ptr, ldb, K2, nv.dptr(dC), N, nv.dptr(dbias), nv.dptr(dZ),
                                    N, epi, split, nv.current_stream()))
    torch.cuda.synchronize()
    assert rel_l2(dC.cpu().numpy(), ref) < TOL


# ----------------------------------------------------------------------------------------------
# not kernel_harness.make_params: its bounds differ (l1 by 1 / sqrt(H), l3 by 0.1)
def make_params(rng, O, A, H, critic):
    I = O + (A if critic else 0)
    u = lambda shp, b: rng.uniform(-b, b, shp)  # noqa: E731
    return {"l1.weight": u((H, I), 1 / np.sqrt(H)), "l1.bias": u((H,), 0.2),
            "l2.weight_ih": u((4 * H, H), 1 / np.sqrt(4 * H) * 2), "l2.weight_hh": u((4 * H, H), 1 / np.sqrt(4 * H) * 2),
            "l2.bias_ih": u((4 * H,), 0.1), "l2.bias_hh": u((4 * H,), 0.1),
            "l3.weight": u((A, H), 0.1), "l3.bias": u((A,), 0.1)}


def flat_params(p):
    return np.concatenate([np.asarray(p[k], np.float32).reshape(-1) for k in lo.PARAM_KEYS])


NET_CASES = [
    # O, A, H, B, T, repeat, critic, first_row
    (5, 2, 32, 4, 7, 1, True, 3),
    (5, 2, 32, 4, 6, 2, False, 0),
    (7, 3, 64, 11, 9, 1, True, 0),
    (7, 3, 64, 11, 5, 2, False, 0),
    (24, 6, 128, 32, 12, 1, True, 4),
    (24, 6, 128, 20, 8, 2, False, 0),
    (17, 6, 256, 40, 10, 1, True, 5),
    (17, 6, 256, 24, 6, 2, False, 0),
    (17, 6, 256, 150, 5, 1, False, 2),      # several clusters, ragged last tile
    (17, 6, 256, 300, 4, 1, True, 1),       # more rows than one wave of NB=16 clusters -> NB=32 tiles
    (3, 1, 128, 9, 6, 1, True, 0),          # Pendulum shape, A = 1
    (6, 2, 96, 5, 4, 1, True, 1),           # generic scan path (H not covered by the cluster kernels)
    (6, 2, 96, 5, 3, 2, False, 0),
    (20, 4, 512, 12, 5, 1, True, 1),        # H = 512: cluster of 16 CTAs, one 16-row tile
    (20, 4, 512, 40, 4, 2, False, 0),       # three clusters of 16 rows (ragged), double actor step
    (376, 17, 512, 150, 3, 1, True, 1),     # cfg-3 widths, more rows than 8 resident clusters x 16 -> 32-row tiles
    (33, 5, 512, 300, 3, 2, False, 0),      # 32-row tiles in two waves of clusters, repeat = 2
    (12, 3, 512, 600, 2, 1, True, 0),       # more rows than one wave of 7 x 80 (forward: 8 clusters of 75 in two waves;
                                            # BPTT: full waves of 32-row clusters + a remainder launch of 16-row clusters)
]


@pytest.fixture(params=["tc", "mma"])
def scan_impl(request, nv):
    """Run the chain tests on both scan implementations: the persistent cluster kernels (default; the hidden sizes they
    do not cover fall through to the per-step path) and the per-step path (one GEMM + one cell kernel per step)."""
    lib = nv.lib()
    lib.r2d2_set_scan_impl(1 if request.param == "tc" else 0)
    yield request.param
    status = scan_status(nv)
    lib.r2d2_set_scan_impl(1)
    assert status == 0, f"a bounded mbarrier wait timed out inside a scan kernel (code {status})"


@pytest.mark.parametrize("O,A,H,B,T,repeat,critic,first_row", NET_CASES)
def test_net_forward_backward(nv, scan_impl, O, A, H, B, T, repeat, critic, first_row):
    rng = np.random.default_rng(O * 1000 + H + B)
    p = make_params(rng, O, A, H, critic)
    obs = rng.standard_normal((T, B, O))
    act = rng.uniform(-1, 1, (T, B, A))
    h0, c0 = 0.3 * rng.standard_normal((B, H)), 0.3 * rng.standard_normal((B, H))
    x = np.concatenate((obs, act), 2) if critic else obs
    p32 = {k: np.asarray(v, np.float32).astype(np.float64) for k, v in p.items()}
    f = lambda a: np.asarray(a, np.float32).astype(np.float64)  # noqa: E731
    sv = lo.net_forward(p32, f(x), f(h0), f(c0), critic=critic, repeat=repeat)
    out_ref = sv["out"][repeat - 1::repeat][first_row:]           # output after the last step of each row
    d_out_rows = rng.standard_normal(out_ref.shape)
    d_out_full = np.zeros_like(sv["out"])
    d_out_full[repeat - 1::repeat][first_row:] = f(d_out_rows)
    g_ref, dx_ref, aux = lo.net_backward(p32, sv, d_out_full, critic=critic, want_wgrad=True, want_dx=True)

    shape = nv.NetShape(O, A, H, int(critic))
    lib = nv.lib()
    npar = lib.r2d2_net_param_count(nv.byref(shape))
    assert npar == flat_params(p).size
    ws = torch.zeros(lib.r2d2_net_workspace_floats(nv.byref(shape), T, B, repeat), device="cuda")
    dparams, dobs, dact = dev(flat_params(p)), dev(obs), dev(act)
    dh0, dc0 = dev(h0), dev(c0)
    out = torch.zeros(((T - first_row), B, A), device="cuda")
    nv.check(lib.r2d2_lstm_net_forward(nv.byref(shape), nv.dptr(dparams), nv.dptr(dobs),
                                       nv.dptr(dact) if critic else None, nv.dptr(dh0), nv.dptr(dc0), T, B, repeat,
                                       first_row, nv.dptr(out), nv.dptr(ws), nv.current_stream()))
    torch.cuda.synchronize()
    assert rel_l2(out.cpu().numpy(), out_ref) < TOL
    grads = torch.zeros(npar, device="cuda")
    d_act = torch.zeros((T, B, A), device="cuda") if critic else None
    d_out_dev = dev(d_out_rows)
    nv.check(lib.r2d2_lstm_net_backward(nv.byref(shape), nv.dptr(dparams), nv.dptr(dobs),
                                        nv.dptr(dact) if critic else None, nv.dptr(d_out_dev), T, B, repeat,
                                        first_row, nv.dptr(grads), nv.dptr(d_act), nv.dptr(ws), nv.current_stream()))
    torch.cuda.synchronize()
    g = grads.cpu().numpy()
    off = 0
    for k in lo.PARAM_KEYS:
        n = g_ref[k].size
        assert rel_l2(g[off:off + n], g_ref[k]) < 5e-5, k
        off += n
    if critic:
        assert rel_l2(d_act.cpu().numpy(), dx_ref[:, :, O:]) < 5e-5


def test_zero_state_matches_explicit_zeros(nv):
    O, A, H, B, T = 5, 2, 64, 6, 4
    rng = np.random.default_rng(3)
    p = make_params(rng, O, A, H, False)
    shape = nv.NetShape(O, A, H, 0)
    lib = nv.lib()
    ws = torch.zeros(lib.r2d2_net_workspace_floats(nv.byref(shape), T, B, 1), device="cuda")
    dparams, dobs = dev(flat_params(p)), dev(rng.standard_normal((T, B, O)))
    outs = []
    for h0 in (None, torch.zeros((B, H), device="cuda")):
        out = torch.zeros((T, B, A), device="cuda")
        nv.check(lib.r2d2_lstm_net_forward(nv.byref(shape), nv.dptr(dparams), nv.dptr(dobs), None, nv.dptr(h0),
                                           nv.dptr(h0), T, B, 1, 0, nv.dptr(out), nv.dptr(ws), nv.current_stream()))
        torch.cuda.synchronize()
        outs.append(out.cpu().numpy())
    assert np.array_equal(outs[0], outs[1])


# ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("L,B,A,Bn,n", [(40, 32, 6, 20, 5), (10, 4, 2, 6, 3), (80, 256, 6, 40, 5), (7, 33, 1, 0, 1),
                                        (80, 512, 17, 40, 5), (5, 1, 3, 2, 2)])
def test_td_priority(nv, L, B, A, Bn, n):
    rng = np.random.default_rng(L * B + A)
    T = Bn + L + n
    q, qn = rng.standard_normal((L, B, A)) * 2, rng.standard_normal((L, B, A)) * 5
    rew = rng.standard_normal((T, B)) * 3
    term = (rng.uniform(size=(T, B)) < 0.1).astype(np.float64)
    f = lambda a: np.asarray(a, np.float32).astype(np.float64)  # noqa: E731
    y, loss, dq, td_sq, prio = lo.td_targets_and_priorities(f(q), f(qn), f(rew), f(term), burn_in=Bn, learning=L,
                                                            n_step=n, gamma=0.997)
    o = {k: torch.zeros(s, device="cuda") for k, s in (("y", (L, B, A)), ("dq", (L, B, A)), ("td", (L, B)),
                                                        ("p", (B,)), ("loss", (1,)))}
    dq_, dqn_, drew_, dterm_ = dev(q), dev(qn), dev(rew), dev(term)   # keep alive across the async launch
    nv.check(nv.lib().r2d2_td_priority(nv.dptr(dq_), nv.dptr(dqn_), nv.dptr(drew_), nv.dptr(dterm_), L, B,
                                       A, Bn, n, 0.997, 0.9, nv.dptr(o["y"]), nv.dptr(o["dq"]), nv.dptr(o["td"]),
                                       nv.dptr(o["p"]), nv.dptr(o["loss"]), nv.current_stream()))
    torch.cuda.synchronize()
    assert rel_l2(o["y"].cpu().numpy(), y) < 1e-6
    assert rel_l2(o["dq"].cpu().numpy(), dq) < 1e-5
    assert rel_l2(o["td"].cpu().numpy(), td_sq) < 1e-5
    assert rel_l2(o["p"].cpu().numpy(), prio) < 1e-5
    assert abs(o["loss"].item() - loss) < 1e-5 * abs(loss)


def test_adam_matches_torch(nv):
    n = 100003
    g = torch.Generator().manual_seed(0)
    p0 = torch.randn(n, generator=g)
    ref_p = p0.clone().requires_grad_(True)
    opt = torch.optim.Adam([ref_p], lr=1e-3)
    p, m, v = p0.clone().cuda(), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    for step in range(1, 6):
        grad = torch.randn(n, generator=g) * (0.1 ** step)
        ref_p.grad = grad.clone()
        opt.step()
        g2 = (2 * grad).cuda()
        nv.check(nv.lib().r2d2_adam_step(nv.dptr(p), nv.dptr(g2), nv.dptr(m), nv.dptr(v), n, step, 1e-3,
                                         0.9, 0.999, 1e-8, 0.5, nv.current_stream()))
    torch.cuda.synchronize()
    assert rel_l2(p.cpu().numpy() - p0.numpy(), ref_p.detach().numpy() - p0.numpy()) < 1e-5

"""Bits of the wgmma GEMM (gemm_packed_kernel), called through the C ABI with the wgmma path selected for every shape.
The cases cover the cfg-3 learner products at full size (gin, dgin, dW_hh), grids of fewer 128 x 128 output tiles
than SMs and of many waves, ragged M, N and K, and every epilogue r2d2_gemm_f32 reaches (bias, tanh, dtanh, add-Z,
split-K).  A chain forward (r2d2_lstm_net_forward at H = 512) adds the b_ih + b_hh epilogue and the z1 operand image.
Each product is checked against a float64 oracle and its SHA-256 against tests/golden/gemm_digests.json.  A change to
how the GEMM schedules its work that keeps every output element's summation order must keep these bits.

  python tools/record_gemm_digests.py PATH   # digests of the library R2D2_B200_LIB points at
"""
import hashlib
import json
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conftest import GOLDEN  # noqa: E402
from kernel_harness import nv  # noqa: E402,F401

pytestmark = pytest.mark.gpu

TOL = 2e-5   # tests/test_gpu_kernels.py::test_gemm (K <= 30720)
# cfg3_dwhh contracts over K = 81920: the fp32 accumulation of that many products alone puts the relative L2 error near
# 6e-5.  Its digest still pins the bits to those of the previous kernel.
TOL_LONG_K = 1e-4
DIGESTS = os.path.join(GOLDEN, "gemm_digests.json")

CASES = {
    # name: layout (0 NT, 1 NN, 2 TN), M, N, K, bias, epilogue (0 none, 1 tanh, 2 dtanh, 3 add-Z), split_k.
    # tiles = ceil(M / 128) * ceil(N / 128) * slices, against 132 SMs
    "cfg3_gin": (0, 64000, 2048, 512, True, 0, 1),          # 8000 tiles
    "cfg3_dgin": (1, 64000, 512, 2048, False, 2, 1),        # 2000 tiles
    "cfg3_dwhh": (2, 2048, 512, 81920, False, 0, 5),        # 320 tiles, 512 k tiles each
    "few_units": (0, 1000, 640, 300, True, 1, 1),           # 40 tiles
    "odd_units": (0, 6784, 640, 256, True, 0, 1),           # 265 tiles: two waves and one more tile
    "three_per_cta": (1, 12667, 512, 256, False, 2, 1),     # 396 tiles: three full waves, ragged M
    "ragged_add_z": (0, 1301, 333, 77, True, 3, 1),
    "ragged_nn": (1, 1301, 333, 77, False, 0, 1),
    "ragged_split_k": (2, 333, 201, 5000, False, 0, 7),
}
# actor chain forward (z1 = tanh(l1(obs)) with its operand image, gin with b_ih + b_hh): obs, act, hidden, T, B
NET_CASES = {"actor_h512": (376, 17, 512, 12, 64)}


def _rel_l2(a, ref):
    """relative L2 error (conftest.rel_l2), on the device: the full-size cases have 10^8 elements"""
    import torch
    return float(torch.linalg.norm(a.double() - ref) / torch.linalg.norm(ref))


def _sha(t):
    return hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).hexdigest()


def run_case(nv, name):
    """returns (C on the device, float64 oracle on the device) of CASES[name]"""
    import torch
    layout, M, N, K, bias, epi, split = CASES[name]
    g = torch.Generator(device="cuda").manual_seed(sum(map(ord, name)))
    shape_a = (K, M) if layout == 2 else (M, K)
    shape_b = (N, K) if layout == 0 else (K, N)
    A = torch.randn(shape_a, device="cuda", generator=g)
    B = torch.randn(shape_b, device="cuda", generator=g)
    bv = torch.randn(N, device="cuda", generator=g) if bias else None
    Z = torch.rand((M, N), device="cuda", generator=g) * 1.8 - 0.9 if epi in (2, 3) else None
    C = torch.zeros((M, N), device="cuda")
    lda, ldb = shape_a[1], shape_b[1]
    lib = nv.lib()
    lib.r2d2_set_gemm_impl(2)   # wgmma path for every shape
    try:
        nv.check(lib.r2d2_gemm_f32(layout, M, N, K, nv.dptr(A), lda, nv.dptr(B), ldb, None, 0, None, 0, 0, nv.dptr(C), N,
                                   nv.dptr(bv), nv.dptr(Z), N, epi, split, nv.current_stream()))
    finally:
        lib.r2d2_set_gemm_impl(1)
    A64, B64 = A.double(), B.double()
    ref = (A64 @ B64.T) if layout == 0 else (A64 @ B64 if layout == 1 else A64.T @ B64)
    if bias:
        ref += bv.double()
    if epi == 1:
        ref = torch.tanh(ref)
    elif epi == 2:
        ref *= 1 - Z.double() ** 2
    elif epi == 3:
        ref += Z.double()
    torch.cuda.synchronize()
    return C, ref


def run_net_case(nv, name):
    """forward of an actor chain through r2d2_lstm_net_forward: returns z1, the gin region, the z1 operand image (all
    device tensors) and the float64 oracle of z1.  The gin region holds gin = z1 W_ih^T + b_ih + b_hh until the scan
    writes the gate activations over it, so its digest covers both."""
    import ctypes
    import torch
    O, A, H, T, B = NET_CASES[name]
    shape = nv.NetShape(O, A, H, 0)
    n_par = nv.lib().r2d2_net_param_count(ctypes.byref(shape))
    ws_floats = nv.lib().r2d2_net_workspace_floats(ctypes.byref(shape), T, B, 1)
    g = torch.Generator(device="cuda").manual_seed(5)
    params = torch.rand(n_par, device="cuda", generator=g) * 0.2 - 0.1
    obs = torch.randn((T * B, O), device="cuda", generator=g)
    h0, c0 = torch.zeros((B, H), device="cuda"), torch.zeros((B, H), device="cuda")
    ws = torch.zeros(ws_floats, device="cuda")
    nv.check(nv.lib().r2d2_lstm_net_forward(ctypes.byref(shape), nv.dptr(params), nv.dptr(obs), None, nv.dptr(h0),
                                            nv.dptr(c0), T, B, 1, 0, None, nv.dptr(ws), nv.current_stream()))
    torch.cuda.synchronize()
    TB, al = T * B, lambda n: (n + 63) // 64 * 64   # noqa: E731  (ChainWs::carve: z1, gin first, z1 image last)
    z1, gin = ws[:TB * H].view(TB, H), ws[al(TB * H):al(TB * H) + TB * 4 * H].view(TB, 4 * H)
    img_floats = al((TB + 127) // 128 * 128 * H)
    img = ws[ws_floats - img_floats:]
    w1, b1 = params[:H * O].view(H, O), params[H * O:H * O + H]   # NetParams::from_flat
    z1_ref = torch.tanh(obs.double() @ w1.double().T + b1.double())
    return z1, gin, img, z1_ref


def digests(nv):
    out = {}
    for name in sorted(CASES):
        C, _ = run_case(nv, name)
        out[name] = _sha(C)
    for name in sorted(NET_CASES):
        z1, gin, img, _ = run_net_case(nv, name)
        out[name] = {"z1": _sha(z1), "gin": _sha(gin), "z1_image": _sha(img)}
    return out


@pytest.fixture(scope="module")
def golden():
    with open(DIGESTS) as f:
        return json.load(f)


@pytest.mark.parametrize("name", sorted(CASES))
def test_gemm_matches_oracle_and_golden_bits(nv, golden, name):
    C, ref = run_case(nv, name)
    assert _rel_l2(C, ref) < (TOL_LONG_K if CASES[name][3] > 32768 else TOL)
    assert _sha(C) == golden[name], "GEMM bits differ from the recorded ones"


@pytest.mark.parametrize("name", sorted(NET_CASES))
def test_chain_forward_matches_oracle_and_golden_bits(nv, golden, name):
    z1, gin, img, z1_ref = run_net_case(nv, name)
    assert _rel_l2(z1, z1_ref) < TOL
    assert {"z1": _sha(z1), "gin": _sha(gin), "z1_image": _sha(img)} == golden[name]


def test_side_stream_input_projections_give_identical_bits(nv):
    """The learner issues some input projections on a low-priority stream beside the persistent scans.  With that stream
    disabled (R2D2_OVERLAP_INPUTS=0) the same products run on the main stream; a seeded run must give the same bits
    either way."""
    import torch
    from oracle import ref_port
    from r2d2_b200 import engine
    kw = dict(obs=40, act=4, hidden=256, batch=64, burn_in=8, learning=16, n_step=3)
    pc, cfg = ref_port.PathConfig(**kw), engine.PathConfig(**kw)
    batches = [ref_port.synthetic_batch(pc, seed=70 + it) for it in range(3)]

    def run(overlap):
        old = os.environ.get("R2D2_OVERLAP_INPUTS")
        os.environ["R2D2_OVERLAP_INPUTS"] = overlap
        try:
            eng = engine.LearnerEngine(cfg, seed=9)
        finally:
            if old is None:
                del os.environ["R2D2_OVERLAP_INPUTS"]
            else:
                os.environ["R2D2_OVERLAP_INPUTS"] = old
        for b in batches:
            eng.set_batch(b)
            eng.step()
        torch.cuda.synchronize()
        out = {k: getattr(eng, k).clone() for k in ("q_value", "target_q_value", "priority", "losses")}
        out.update({net: eng.flat[net].clone() for net in ("actor", "critic")})
        eng.close()
        return out

    side, main = run("1"), run("0")
    for k in side:
        assert torch.equal(side[k], main[k]), k

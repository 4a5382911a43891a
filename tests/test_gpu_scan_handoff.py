"""Long chains through the persistent cluster scan kernels, called through the C ABI, against a float64 LSTM
recurrence.  The kernels hand h_t (forward) and the dh partials (BPTT) from CTA to CTA through per-source mbarriers
that are reused every second step, so chains of 125+ steps wrap every barrier phase many times; the batch sizes need
several waves of clusters and leave a ragged last tile.  The same chain run twice must give the same bits."""

import numpy as np
import pytest
import torch

from conftest import rel_l2
from kernel_harness import nv, scan_status  # noqa: F401
from oracle import learner_oracle as lo

pytestmark = pytest.mark.gpu

TOL_FWD, TOL_BWD = 2e-5, 5e-5   # tests/test_gpu_kernels.py: chain outputs / gradients

CASES = [
    # H, B, T, repeat
    (128, 1500, 150, 1),
    (256, 520, 64, 2),
    (512, 456, 125, 1),
    (512, 300, 64, 2),
]


@pytest.mark.parametrize("H,B,T,repeat", CASES)
def test_long_chain_matches_oracle_and_repeats_bitwise(nv, H, B, T, repeat):
    lib = nv.lib()
    lib.r2d2_set_scan_impl(1)
    rng = np.random.default_rng(H * 7 + B + repeat)
    S = T * repeat
    f32 = lambda a: np.asarray(a, np.float32)  # noqa: E731
    gin = f32(0.5 * rng.standard_normal((T, B, 4 * H)))
    whh = f32(rng.uniform(-1, 1, (4 * H, H)) * 2 / np.sqrt(4 * H))
    h0, c0 = f32(0.3 * rng.standard_normal((B, H))), f32(0.3 * rng.standard_normal((B, H)))
    dh_head = f32(rng.standard_normal((T, B, H)))
    ref = lo.lstm_scan(*(a.astype(np.float64) for a in (gin, whh, h0, c0, dh_head)), repeat=repeat)

    d = lambda a: torch.as_tensor(a).cuda()  # noqa: E731
    d_gin, d_whh, d_h0, d_c0, d_dh = d(gin), d(whh), d(h0), d(c0), d(dh_head)
    scratch = torch.empty(B * 4 * H + 64, device="cuda")   # used by the per-step path only
    st = nv.current_stream()
    runs = []
    for _ in range(2):
        gates = torch.empty((S, B, 4 * H), device="cuda")
        hs, cs = torch.empty((S + 1, B, H), device="cuda"), torch.empty((S + 1, B, H), device="cuda")
        dgates = torch.empty_like(gates)
        dgin = torch.empty((T, B, 4 * H), device="cuda") if repeat > 1 else dgates
        nv.check(lib.r2d2_lstm_scan_forward(nv.dptr(d_gin), nv.dptr(d_whh), nv.dptr(d_h0), nv.dptr(d_c0), nv.dptr(gates),
                                            nv.dptr(hs), nv.dptr(cs), None, T, B, H, repeat, nv.dptr(scratch), st))
        nv.check(lib.r2d2_lstm_scan_backward(nv.dptr(gates), nv.dptr(hs), nv.dptr(cs), nv.dptr(d_whh), nv.dptr(d_dh), 0,
                                             nv.dptr(dgates), nv.dptr(dgin), T, B, H, repeat, nv.dptr(scratch), st))
        torch.cuda.synchronize()
        runs.append((hs.cpu().numpy(), dgin.cpu().numpy()))
    status = scan_status(nv, st)
    assert status == 0, f"a bounded hand-off wait expired inside a scan kernel (code {status})"

    (hs_a, dgin_a), (hs_b, dgin_b) = runs
    assert np.array_equal(hs_a, hs_b) and np.array_equal(dgin_a, dgin_b), "two runs of the same chain differ"
    assert rel_l2(hs_a[1:], ref["hs"][1:]) < TOL_FWD
    assert rel_l2(dgin_a, ref["dgin"]) < TOL_BWD

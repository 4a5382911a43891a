"""BPTT cluster scan with the per-step activation stage (gates, c_prev and dh_head of step s-1 copied into shared memory
while step s runs), called through the C ABI.  The chains cover the batch tiles the dispatcher picks (NB = 8 and 16 at
H = 512, NB = 32 at H = 256), repeat 1 and 2, steps with and without a dh_head row, a ragged last tile, and dG written
in place over the gates as the learner does.  Each chain is checked against a float64 recurrence, and the SHA-256 of
its dgates / dgin bits against tests/golden/scan_bwd_digests.json: the stage only moves loads, every sum keeps its
order, so the bits must not change.

  python tests/test_gpu_scan_bwd_stage.py --write-digests PATH   # digests of the library R2D2_B200_LIB points at
"""
import hashlib
import json
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conftest import GOLDEN, rel_l2  # noqa: E402
from kernel_harness import nv, scan_status  # noqa: E402,F401
from oracle import learner_oracle as lo  # noqa: E402

pytestmark = pytest.mark.gpu

TOL_FWD, TOL_BWD = 2e-5, 5e-5   # tests/test_gpu_kernels.py: chain outputs / gradients
DIGESTS = os.path.join(GOLDEN, "scan_bwd_digests.json")

CASES = {
    # name: H, B, T, repeat, head_first_step.  The tile is the narrowest whose clusters are all resident on an H100:
    # B <= 40 gives NB = 8 at H = 512, B = 200 gives NB = 16 at H = 512, B = 600 gives NB = 32 at H = 256.
    "h512_nb8_rep1": (512, 37, 48, 1, 9),
    "h512_nb8_rep2": (512, 37, 24, 2, 10),
    "h512_nb16_rep1": (512, 200, 48, 1, 9),
    "h512_nb16_rep2": (512, 200, 24, 2, 10),
    "h256_nb32_rep1": (256, 600, 48, 1, 9),
    "h256_nb32_rep2": (256, 600, 24, 2, 10),
}


def inputs(H, B, T, repeat, head_first_step):
    rng = np.random.default_rng(H * 131 + B * 7 + repeat)
    f32 = lambda a: np.asarray(a, np.float32)  # noqa: E731
    gin = f32(0.5 * rng.standard_normal((T, B, 4 * H)))
    whh = f32(rng.uniform(-1, 1, (4 * H, H)) * 2 / np.sqrt(4 * H))
    h0, c0 = f32(0.3 * rng.standard_normal((B, H))), f32(0.3 * rng.standard_normal((B, H)))
    dh_head = f32(rng.standard_normal(((T * repeat - head_first_step) // repeat, B, H)))
    return gin, whh, h0, c0, dh_head


def run_chain(nv, H, B, T, repeat, head_first_step):
    """forward + BPTT through the cluster kernels; dG overwrites the gates.  Returns hs, dgates, dgin (host arrays)."""
    import torch
    lib = nv.lib()
    lib.r2d2_set_scan_impl(1)
    gin, whh, h0, c0, dh_head = inputs(H, B, T, repeat, head_first_step)
    S = T * repeat
    d = lambda a: torch.as_tensor(a).cuda()  # noqa: E731
    d_gin, d_whh, d_h0, d_c0, d_dh = d(gin), d(whh), d(h0), d(c0), d(dh_head)
    scratch = torch.empty(B * 4 * H + 64, device="cuda")   # used by the per-step path only
    st = nv.current_stream()
    gates = torch.empty((S, B, 4 * H), device="cuda")
    hs, cs = torch.empty((S + 1, B, H), device="cuda"), torch.empty((S + 1, B, H), device="cuda")
    dgin = torch.empty((T, B, 4 * H), device="cuda") if repeat > 1 else gates
    nv.check(lib.r2d2_lstm_scan_forward(nv.dptr(d_gin), nv.dptr(d_whh), nv.dptr(d_h0), nv.dptr(d_c0), nv.dptr(gates),
                                        nv.dptr(hs), nv.dptr(cs), None, T, B, H, repeat, nv.dptr(scratch), st))
    nv.check(lib.r2d2_lstm_scan_backward(nv.dptr(gates), nv.dptr(hs), nv.dptr(cs), nv.dptr(d_whh), nv.dptr(d_dh),
                                         head_first_step, nv.dptr(gates), nv.dptr(dgin), T, B, H, repeat,
                                         nv.dptr(scratch), st))
    torch.cuda.synchronize()
    return hs.cpu().numpy(), gates.cpu().numpy(), dgin.cpu().numpy()


def digests(dgates, dgin):
    return {"dgates": hashlib.sha256(np.ascontiguousarray(dgates).tobytes()).hexdigest(),
            "dgin": hashlib.sha256(np.ascontiguousarray(dgin).tobytes()).hexdigest()}


@pytest.fixture(scope="module")
def golden():
    with open(DIGESTS) as f:
        return json.load(f)


@pytest.mark.parametrize("name", sorted(CASES))
def test_bwd_stage_matches_oracle_and_golden_bits(nv, golden, name):
    H, B, T, repeat, hfs = CASES[name]
    hs, dgates, dgin = run_chain(nv, H, B, T, repeat, hfs)
    assert scan_status(nv) == 0, "a bounded hand-off wait expired inside a scan kernel"
    ref = lo.lstm_scan(*(a.astype(np.float64) for a in inputs(H, B, T, repeat, hfs)), repeat=repeat,
                       head_first_step=hfs)
    assert rel_l2(hs[1:], ref["hs"][1:]) < TOL_FWD
    assert rel_l2(dgin, ref["dgin"]) < TOL_BWD
    assert digests(dgates, dgin) == golden[name], "BPTT bits differ from the recorded ones"


if __name__ == "__main__":
    if len(sys.argv) != 3 or sys.argv[1] != "--write-digests":
        raise SystemExit(__doc__)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path[:0] = [root, os.path.join(root, "pytorch-r2d2-dpg_b200")]
    from r2d2_b200 import native
    out = {}
    for name, (H, B, T, repeat, hfs) in sorted(CASES.items()):
        _, dgates, dgin = run_chain(native, H, B, T, repeat, hfs)
        assert scan_status(native) == 0, name
        out[name] = digests(dgates, dgin)
        print(name, out[name])
    with open(sys.argv[2], "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")

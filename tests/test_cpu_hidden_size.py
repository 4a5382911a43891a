"""CPU checks behind tests/test_gpu_hidden_size.py: the float64 scan oracle (oracle/learner_oracle.lstm_scan) against
torch.nn.LSTMCell and autograd, and the two localised error bounds (tile_err, unit_group_err) against errors that a
whole-tensor relative L2 norm dilutes below its bound."""
import numpy as np
import pytest
import torch

from conftest import rel_l2
from learner_harness import tile_err, unit_group_err
from oracle import learner_oracle as lo


def _autograd_scan(gin, whh, h0, c0, dh_head, repeat, head_first_step):
    """The same recurrence through torch.nn.LSTMCell in float64 (gin enters as the input projection with W_ih = I and
    zero biases), dh_head as the gradient of sum(dh_head * h) at the head steps; gradients by autograd."""
    T, B, H4 = gin.shape
    H, S = H4 // 4, T * repeat
    cell = torch.nn.LSTMCell(H4, H).double()
    with torch.no_grad():
        cell.weight_ih.copy_(torch.eye(H4, dtype=torch.float64))
        cell.weight_hh.copy_(torch.as_tensor(whh))
        cell.bias_ih.zero_()
        cell.bias_hh.zero_()
    x = torch.tensor(gin, requires_grad=True)
    h = torch.zeros(B, H, dtype=torch.float64) if h0 is None else torch.as_tensor(h0)
    c = torch.zeros(B, H, dtype=torch.float64) if c0 is None else torch.as_tensor(c0)
    hs, cs, head_in, loss = [h], [c], [], 0.0
    for s in range(S):
        h, c = cell(x[s // repeat], (h, c))
        hs.append(h)
        cs.append(c)
        if s % repeat == repeat - 1:
            head_in.append(torch.tanh(h))
        rel = s - head_first_step
        if rel >= 0 and rel % repeat == repeat - 1:
            loss = loss + (torch.as_tensor(dh_head[rel // repeat]) * h).sum()
    loss.backward()
    return (torch.stack(hs).detach().numpy(), torch.stack(cs).detach().numpy(), torch.stack(head_in).detach().numpy(),
            x.grad.numpy())


@pytest.mark.parametrize("H,B,T,repeat,hfs,zero_state", [(8, 3, 5, 1, 0, False), (12, 4, 4, 2, 3, True),
                                                          (32, 5, 6, 2, 0, False), (20, 2, 7, 1, 4, True)])
def test_scan_oracle_matches_lstm_cell_autograd(H, B, T, repeat, hfs, zero_state):
    rng = np.random.default_rng(H * 10 + B)
    gin = 0.5 * rng.standard_normal((T, B, 4 * H))
    whh = rng.uniform(-1, 1, (4 * H, H)) * 2 / np.sqrt(4 * H)
    h0, c0 = (None, None) if zero_state else (0.3 * rng.standard_normal((B, H)), 0.3 * rng.standard_normal((B, H)))
    dh_head = rng.standard_normal(((T * repeat - hfs) // repeat, B, H))
    ref = lo.lstm_scan(gin, whh, h0, c0, dh_head, repeat=repeat, head_first_step=hfs)
    hs, cs, head_in, dgin = _autograd_scan(gin, whh, h0, c0, dh_head, repeat, hfs)
    for name, got, want in (("hs", ref["hs"], hs), ("cs", ref["cs"], cs), ("head_in", ref["head_in"], head_in),
                            ("dgin", ref["dgin"], dgin)):
        assert got.shape == want.shape, name
        assert rel_l2(got, want) < 1e-12, name
    # post-activation gates from the states: c_{s+1} = f c_s + i g, h_{s+1} = o tanh(c_{s+1})
    i, f, g, o = np.split(ref["gates"], 4, axis=2)
    assert rel_l2(f * ref["cs"][:-1] + i * g, cs[1:]) < 1e-12
    assert rel_l2(o * np.tanh(ref["cs"][1:]), hs[1:]) < 1e-12
    assert rel_l2(ref["dgates"].reshape(T, repeat, B, 4 * H).sum(1), dgin) < 1e-12


def _perturbed(shape, where, seed):
    """ref ~ N(0, 1) and x = ref with a relative error of 1e-4 on the elements `where`."""
    rng = np.random.default_rng(seed)
    ref = rng.standard_normal(shape)
    x = ref.copy()
    x[where] *= 1.0 + 1e-4 * np.sign(rng.standard_normal(x[where].shape))
    return x, ref


@pytest.mark.parametrize("B,NB", [(1500, 32), (4099, 8), (600, 16)])
def test_tile_err_finds_an_error_in_one_tile(B, NB):
    last = (B - 1) // NB * NB                                   # the ragged last tile
    for rows in (slice(NB, 2 * NB), slice(last, B)):
        x, ref = _perturbed((6, B, 64), (slice(None), rows), seed=B + NB)
        assert rel_l2(x, ref) < 2e-5
        assert tile_err(x, ref, NB) == pytest.approx(1e-4, rel=1e-6)
    assert tile_err(ref, ref, NB) == 0.0


# 4H axes at H = 512 / 256 have 64 / 32 groups: rel_l2 dilutes the error below 2e-5.  At H = 512 on an H axis (16
# groups) and at H = 20 (one short group) the dilution is smaller, but the group bound is the same.
@pytest.mark.parametrize("H,four", [(512, True), (256, True), (512, False), (20, False)])
def test_unit_group_err_finds_an_error_in_one_unit_group(H, four):
    n = 4 * H if four else H
    start = 2 * H + 32 if four else 32 * ((H // 32) // 2)        # one 32-unit group (of gate block g on a 4H axis)
    x, ref = _perturbed((12, 40, n), (slice(None), slice(None), slice(start, min(start + 32, n))), seed=H)
    if four:
        assert rel_l2(x, ref) < 2e-5
    assert unit_group_err(x, ref, H) == pytest.approx(1e-4, rel=1e-6)
    assert unit_group_err(ref, ref, H) == 0.0
    if four:   # groups are taken per gate block: the last unit of block i is in a group of block i's units only
        y = ref.copy()
        y[..., H - 1] += 1.0
        assert unit_group_err(y, ref, H) == pytest.approx(
            np.linalg.norm(y[..., H - 32:H] - ref[..., H - 32:H]) / np.linalg.norm(ref[..., H - 32:H]))

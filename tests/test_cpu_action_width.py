"""Pin the float64 oracle (oracle/learner_oracle.py) against the torch port of the reference (oracle/ref_port.py) at wide
action spaces.  The GPU tests of tests/test_gpu_action_width.py trust both at A = 12 .. 64; the reference goldens stop at
A = 6.  Reduced sizes of the learner shapes used there, two consecutive iterations each (Adam state carried), with the
bounds of test_oracle_golden.py::test_numpy_oracle_matches_port_on_edge_shapes.  Every output with an action axis is
also bounded per action column (col_err), so that one wrong column cannot hide in the norm of the whole tensor."""
import numpy as np
import pytest
import torch

from conftest import rel_l2
from learner_harness import col_err
from oracle import learner_oracle as lo
from oracle import ref_port


def action_views(block, O, A):
    """The action-indexed parts of a parameter / gradient dict as [-1, A] arrays: l3.weight rows, l3.bias, and the
    action columns of the critic's l1.weight (None for the actor)."""
    out = {"l3.weight": np.asarray(block["l3.weight"]).T, "l3.bias": np.asarray(block["l3.bias"])}
    if np.asarray(block["l1.weight"]).shape[1] == O + A:
        out["l1.weight[:, O:]"] = np.asarray(block["l1.weight"])[:, O:]
    return out


CASES = [
    # obs, act, hidden, batch, burn_in, learning, n_step: reduced sizes of the GPU learner shapes
    (8, 24, 32, 3, 2, 4, 3),      # the largest A on the GPU's two-pass TD route, O + A = 32
    (7, 25, 32, 3, 2, 3, 2),      # first A on the column TD kernel
    (24, 38, 64, 4, 2, 4, 2),     # dog-sized action space, O + A = 62
    (17, 12, 64, 2, 3, 5, 3),     # A between the thin-kernel buckets
    (67, 64, 64, 2, 2, 3, 2),     # the policy step's maximum A
]


@pytest.mark.parametrize("obs,act,hidden,batch,burn_in,learning,n_step", CASES)
def test_numpy_oracle_matches_port_at_wide_action_spaces(obs, act, hidden, batch, burn_in, learning, n_step):
    torch.set_num_threads(1)
    pc = ref_port.PathConfig(obs=obs, act=act, hidden=hidden, batch=batch, burn_in=burn_in, learning=learning,
                             n_step=n_step)
    port = ref_port.PortLearner(pc, seed=23)
    sd = lambda m: {k: v.detach().numpy().copy() for k, v in m.state_dict().items()}  # noqa: E731
    ol = lo.OracleLearner(sd(port.actor), sd(port.critic), burn_in=burn_in, learning=learning, n_step=n_step)
    A = act
    for it in range(2):
        batch_np = ref_port.synthetic_batch(pc, seed=200 + it)
        ref = port.iteration(batch_np)
        out = ol.iteration(batch_np)
        for k in ("q_value", "target_q_value"):
            assert rel_l2(out[k], ref[k]) < 5e-5, (it, k)
            assert col_err(out[k], ref[k], A) < 5e-5, (it, k)
        assert rel_l2(out["priority"], ref["priority"]) < 5e-5
        assert abs(out["critic_loss"] - ref["critic_loss"]) < 1e-4 * abs(ref["critic_loss"]) + 1e-9
        assert abs(out["actor_loss"] - ref["actor_loss"]) < 1e-4 * abs(ref["actor_loss"]) + 1e-9
        for net in ("actor", "critic"):
            for k in lo.PARAM_KEYS:
                assert rel_l2(out[f"{net}_grad"][k], ref[f"{net}_grad"][k]) < 5e-4, (it, net, k)
            got, want = action_views(out[f"{net}_grad"], obs, A), action_views(ref[f"{net}_grad"], obs, A)
            for k in want:
                assert col_err(got[k], want[k], A) < 5e-4, (it, net, k)

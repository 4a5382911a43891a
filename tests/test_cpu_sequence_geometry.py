"""CPU checks behind tests/test_gpu_sequence_geometry.py: the float64 oracle (oracle/learner_oracle.py) against the torch
port of the reference (oracle/ref_port.py) at the windows the GPU module runs and the goldens never do (burn-in 0,
n-step 1, n-step longer than the learning window, batch 1); the one-step window (L = 1), which neither the reference's
priority nor the oracle's defines and PathConfig refuses; and the per-time-row error bound step_err."""
import numpy as np
import pytest
import torch

from conftest import rel_l2
from learner_harness import step_err
from oracle import learner_oracle as lo
from oracle import ref_port

# obs, act, hidden, batch, burn_in, learning, n_step
WINDOWS = [(5, 2, 16, 1, 0, 2, 1), (6, 3, 16, 2, 0, 8, 5), (4, 2, 16, 3, 1, 3, 1), (5, 2, 16, 2, 2, 2, 10),
           (7, 3, 32, 1, 0, 9, 12)]


@pytest.mark.parametrize("obs,act,hidden,batch,burn_in,learning,n_step", WINDOWS)
def test_oracle_matches_port_at_edge_windows(obs, act, hidden, batch, burn_in, learning, n_step):
    torch.set_num_threads(1)
    pc = ref_port.PathConfig(obs=obs, act=act, hidden=hidden, batch=batch, burn_in=burn_in, learning=learning,
                             n_step=n_step)
    port = ref_port.PortLearner(pc, seed=31)
    sd = lambda m: {k: v.detach().numpy().copy() for k, v in m.state_dict().items()}  # noqa: E731
    ol = lo.OracleLearner(sd(port.actor), sd(port.critic), burn_in=burn_in, learning=learning, n_step=n_step)
    for it in range(2):
        batch_np = ref_port.synthetic_batch(pc, seed=300 + it, terminal_frac=0.5)
        ref = port.iteration(batch_np)
        out = ol.iteration(batch_np)
        for k in ("q_value", "target_q_value"):
            assert out[k].shape == ref[k].shape == (learning * batch, act), (it, k)
            assert rel_l2(out[k], ref[k]) < 5e-5, (it, k)
            assert step_err(out[k].reshape(learning, batch, act), ref[k].reshape(learning, batch, act)) < 5e-5, (it, k)
        assert rel_l2(out["priority"], ref["priority"]) < 5e-5
        assert abs(out["critic_loss"] - ref["critic_loss"]) < 1e-4 * abs(ref["critic_loss"]) + 1e-9
        assert abs(out["actor_loss"] - ref["actor_loss"]) < 1e-4 * abs(ref["actor_loss"]) + 1e-9
        for net in ("actor", "critic"):
            for k in lo.PARAM_KEYS:
                assert rel_l2(out[f"{net}_grad"][k], ref[f"{net}_grad"][k]) < 5e-4, (it, net, k)
                assert rel_l2(out[f"{net}_after"][k], ref[f"{net}_after"][k]) < 1e-5, (it, net, k)


def test_one_step_window_has_no_priority_for_the_last_sequence():
    """At L = 1 the [b:-1:B] series of b = B - 1 is empty: the reference's calc_priority takes max([]) and the oracle
    max of an empty array, and both raise rather than define a priority; the other sequences keep theirs."""
    import utils as dropin_utils
    rng = np.random.default_rng(0)
    L, B, A, Bn, n = 1, 3, 2, 0, 1
    q, qn = rng.standard_normal((L, B, A)), rng.standard_normal((L, B, A))
    rew, term = rng.standard_normal((Bn + L + n, B)), np.zeros((Bn + L + n, B))
    with pytest.raises(ValueError):
        lo.td_targets_and_priorities(q, qn, rew, term, burn_in=Bn, learning=L, n_step=n, gamma=0.997)
    td = np.mean((q - rng.standard_normal((L, B, A))) ** 2, axis=2).reshape(-1)
    for b in range(B - 1):
        assert dropin_utils.calc_priority(td[b:-1:B]) == pytest.approx(td[b])
    with pytest.raises(ValueError):
        dropin_utils.calc_priority(td[B - 1:-1:B])
    with pytest.raises(ValueError):
        ref_port.sequence_priority(td[B - 1:-1:B])


@pytest.mark.parametrize("field,value", [("learning", 1), ("learning", 0), ("learning", -3), ("burn_in", -1),
                                         ("n_step", 0), ("n_step", -2), ("learning", 2.0), ("burn_in", True)])
def test_path_config_refuses_bad_windows(field, value):
    from r2d2_b200 import engine
    kw = dict(obs=3, act=2, hidden=16, batch=4, burn_in=2, learning=4, n_step=2)
    with pytest.raises(ValueError, match=field):
        engine.PathConfig(**dict(kw, **{field: value}))


def test_path_config_accepts_edge_windows():
    from r2d2_b200 import engine
    for Bn, L, n in ((0, 2, 1), (0, 2, 10), (80, 400, 5), (np.int64(1), np.int32(3), 1)):
        cfg = engine.PathConfig(obs=3, act=2, burn_in=Bn, learning=L, n_step=n)
        assert cfg.rows == Bn + L + n


def test_step_err_finds_an_error_in_one_time_row():
    """A 1e-4 relative error in one of T = 300 rows: rel_l2 sees it diluted to about 1e-4 / sqrt(300) = 6e-6, under a
    2e-5 bound; step_err reports the 1e-4.  Along a time axis that is not the first one as well."""
    rng = np.random.default_rng(3)
    ref = rng.standard_normal((300, 33, 6))
    for t in (0, 157, 299):
        x = ref.copy()
        x[t] *= 1.0 + 1e-4 * np.sign(rng.standard_normal(x[t].shape))
        assert rel_l2(x, ref) < 2e-5
        assert step_err(x, ref) == pytest.approx(1e-4, rel=1e-6)
        assert step_err(np.moveaxis(x, 0, 1), np.moveaxis(ref, 0, 1), axis=1) == pytest.approx(1e-4, rel=1e-6)
    assert step_err(ref, ref) == 0.0


def test_step_err_measures_a_vanishing_row_against_the_rms_row():
    """A BPTT row far from the head may flush to zero in fp32 where float64 keeps 1e-40: that row is measured against
    1e-3 of the RMS row norm, so it counts as (nearly) exact; an error of that size in a normal row is still seen."""
    rng = np.random.default_rng(4)
    ref = rng.standard_normal((50, 8, 16))
    ref[0] *= 1e-40
    x = ref.copy()
    x[0] = 0.0
    assert step_err(x, ref) < 1e-30
    x[7] += 1e-3 * np.sqrt(np.mean(np.sum(ref.reshape(50, -1) ** 2, axis=1)))
    assert step_err(x, ref) > 1e-4

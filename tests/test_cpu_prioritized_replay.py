"""Prioritized replay on the host side: PathConfig validation, the drop-in modules' environment switches, and the float64
oracle's importance-weighted TD gradient against a finite difference of its loss."""
import sys

import numpy as np
import pytest

from learner_harness import fake_engine_learner
from oracle import learner_oracle as lo
from oracle import ref_port


def test_path_config_exponents_are_validated():
    from r2d2_b200 import engine
    cfg = engine.PathConfig(obs=3, act=1)
    assert (cfg.priority_exponent, cfg.is_exponent) == (1.0, 0.0)       # the reference's behaviour
    engine.PathConfig(obs=3, act=1, priority_exponent=0.0, is_exponent=1.0)
    for bad in ({"priority_exponent": 1.5}, {"priority_exponent": -0.1}, {"is_exponent": 1.01},
                {"is_exponent": -1.0}, {"priority_exponent": float("nan")}):
        with pytest.raises(ValueError):
            engine.PathConfig(obs=3, act=1, **bad)


def test_dropin_environment_switches(monkeypatch, tmp_path):
    lr = fake_engine_learner(monkeypatch, tmp_path, R2D2_PRIORITY_EXPONENT="0.9", R2D2_IS_EXPONENT="0.6")
    assert lr.engine.cfg.priority_exponent == 0.9 and lr.engine.cfg.is_exponent == 0.6
    assert lr.memory.priority_exponent == 0.9 and lr.memory._cfg().priority_exponent == 0.9
    monkeypatch.delenv("R2D2_PRIORITY_EXPONENT")
    monkeypatch.delenv("R2D2_IS_EXPONENT")
    lr = fake_engine_learner(monkeypatch, tmp_path)
    assert (lr.engine.cfg.priority_exponent, lr.engine.cfg.is_exponent) == (1.0, 0.0)
    assert lr.memory._cfg().priority_exponent == 1.0
    with pytest.raises(ValueError):
        fake_engine_learner(monkeypatch, tmp_path, R2D2_PRIORITY_EXPONENT="2")
    with pytest.raises(ValueError):
        fake_engine_learner(monkeypatch, tmp_path, R2D2_IS_EXPONENT="-0.5")


def test_replay_memory_exponent_argument_and_environment(monkeypatch):
    monkeypatch.setenv("R2D2_PRIORITY_EXPONENT", "0.6")
    sys.modules.pop("replay_memory", None)
    import replay_memory as dropin_rm
    try:
        assert dropin_rm.LearnerReplayMemory(batch_size=4).priority_exponent == 0.6
        assert dropin_rm.LearnerReplayMemory(batch_size=4, priority_exponent=0.0)._cfg().priority_exponent == 0.0
        with pytest.raises(ValueError):
            dropin_rm.LearnerReplayMemory(batch_size=4, priority_exponent=1.2)
    finally:
        sys.modules.pop("replay_memory", None)


def test_weighted_td_gradient_matches_finite_difference():
    rng = np.random.default_rng(3)
    Bn, L, n, B, A = 2, 5, 2, 4, 3
    T = Bn + L + n
    q, q_next = rng.standard_normal((L, B, A)), rng.standard_normal((L, B, A))
    rew, term = rng.standard_normal((T, B)), (rng.uniform(size=(T, B)) < 0.2).astype(np.float64)
    w = rng.uniform(0.1, 1.0, B)
    kw = dict(burn_in=Bn, learning=L, n_step=n, gamma=0.997)
    td = lambda *a: lo.td_targets_and_priorities(*a, **kw, is_weight=w)  # noqa: E731
    _, loss, dq, td_sq, prio = td(q, q_next, rew, term)
    _, loss0, dq0, td_sq0, prio0 = lo.td_targets_and_priorities(q, q_next, rew, term, **kw)
    assert np.array_equal(td_sq, td_sq0) and np.array_equal(prio, prio0)      # unweighted by definition
    assert abs(loss - np.sum(w[None, :] * td_sq0) / (L * B)) < 1e-12
    eps = 1e-6
    fd = np.zeros_like(q)
    for idx in np.ndindex(q.shape):
        qp, qm = q.copy(), q.copy()
        qp[idx] += eps
        qm[idx] -= eps
        fd[idx] = (td(qp, q_next, rew, term)[1] - td(qm, q_next, rew, term)[1]) / (2 * eps)
    assert np.abs(fd - dq).max() < 1e-8 * max(1.0, np.abs(dq).max())
    # unit weights are the unweighted loss
    _, loss1, dq1, _, _ = lo.td_targets_and_priorities(q, q_next, rew, term, **kw, is_weight=np.ones(B))
    assert abs(loss1 - loss0) < 1e-14 and np.allclose(dq1, dq0, rtol=1e-14, atol=0)


def test_weighted_iteration_restores_the_unweighted_oracle():
    pc = ref_port.PathConfig(obs=4, act=2, hidden=8, batch=3, burn_in=2, learning=3, n_step=2)
    port = ref_port.PortLearner(pc, seed=1)
    sd = lambda m: {k: v.detach().numpy() for k, v in m.state_dict().items()}  # noqa: E731
    batch = ref_port.synthetic_batch(pc, seed=2)
    a = lo.OracleLearner(sd(port.actor), sd(port.critic), burn_in=2, learning=3, n_step=2)
    b = lo.OracleLearner(sd(port.actor), sd(port.critic), burn_in=2, learning=3, n_step=2)
    ow = a.iteration(dict(batch, is_weight=np.full(3, 0.5)))
    o1 = b.iteration(batch)
    assert abs(ow["critic_loss"] - 0.5 * o1["critic_loss"]) < 1e-12
    for k in lo.PARAM_KEYS:
        assert np.allclose(ow["critic_grad"][k], 0.5 * o1["critic_grad"][k], rtol=1e-10, atol=1e-300)

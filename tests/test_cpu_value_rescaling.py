"""R2D2's n-step target options on the host side: the float64 oracle's h_eps / h_eps^-1 against high-precision decimal
arithmetic, the float32 torch functions of utils.py against the oracle, the drop-in Actor's priorities in every mode
against the float64 actor oracle, validation of PathConfig / the environment variables / checkpoints, and the compiler's
report on every TD and actor-priority kernel instantiation (all present, no spills, no local memory)."""
import decimal
import itertools
import re

import numpy as np
import pytest
import torch

from conftest import rel_l2
from learner_harness import fake_engine_learner
from oracle import actor_oracle
from oracle import learner_oracle as lo
from sass_report import functions, library_sass, ops, ptxas_report

EPS = (0.0, 1e-3, 1e-2)
MODES = [(r, m) for r in ("reference", "invertible") for m in ("squared", "abs")]


def _inputs():
    rng = np.random.default_rng(0)
    mag = 10.0 ** rng.uniform(-8, 6, 3000)
    x = np.concatenate(([0.0, 1e-30, -1e-30, 1e-8, -1e-8, 1e6, -1e6], mag * rng.choice([-1.0, 1.0], mag.size)))
    return x


# ------------------------------------------------------------------------------------------------ 1. oracle vs decimal
def _dec_h(x, eps):
    """Textbook h_eps at 100 significant digits: the cancellation near 0 costs at most ~30 of them."""
    with decimal.localcontext() as ctx:
        ctx.prec = 100
        d, e = decimal.Decimal(float(x)), decimal.Decimal(eps)
        s = 1 if d > 0 else (-1 if d < 0 else 0)
        return s * ((abs(d) + 1).sqrt() - 1) + e * d


def _dec_h_inv(x, eps):
    """The paper's closed form ((sqrt(1 + 4 eps (|x| + 1 + eps)) - 1) / (2 eps))^2 - 1, or (|x| + 1)^2 - 1 at eps = 0."""
    with decimal.localcontext() as ctx:
        ctx.prec = 100
        d, e = decimal.Decimal(float(x)), decimal.Decimal(eps)
        s = 1 if d > 0 else (-1 if d < 0 else 0)
        a = abs(d)
        m = (a + 1) ** 2 - 1 if eps == 0 else (((1 + 4 * e * (a + 1 + e)).sqrt() - 1) / (2 * e)) ** 2 - 1
        return s * m


def _rel(got, want):
    want = float(want)
    return 0.0 if got == want else abs(got - want) / abs(want)


@pytest.mark.parametrize("eps", EPS)
def test_oracle_matches_decimal(eps):
    e64 = float(np.float64(eps))   # the decimal side sees the same binary eps
    worst = {"h": 0.0, "h_inv": 0.0, "round_trip": 0.0}
    for x in _inputs():
        worst["h"] = max(worst["h"], _rel(float(lo.h_eps(x, e64)), _dec_h(x, e64)))
        worst["h_inv"] = max(worst["h_inv"], _rel(float(lo.h_eps_inv(x, e64)), _dec_h_inv(x, e64)))
        worst["round_trip"] = max(worst["round_trip"], _rel(float(lo.h_eps(lo.h_eps_inv(x, e64), e64)), x))
    assert max(worst.values()) < 1e-14, worst
    assert lo.h_eps(0.0, eps) == 0.0 and lo.h_eps_inv(0.0, eps) == 0.0


# ------------------------------------------------------------------------------------------------ 2. float32 utils
@pytest.mark.parametrize("eps", EPS)
def test_float32_utils_match_oracle(eps):
    import utils
    x32 = _inputs().astype(np.float32)
    x = torch.from_numpy(x32)
    e = float(np.float32(eps))     # torch applies the python scalar in float32
    for name, got, want in (("h", utils.value_rescale(x, eps).numpy(), lo.h_eps(x32.astype(np.float64), e)),
                            ("h_inv", utils.inverse_value_rescale(x, eps).numpy(), lo.h_eps_inv(x32.astype(np.float64), e))):
        assert got.dtype == np.float32
        err = np.abs(got - want) / np.maximum(np.abs(want), 1e-300)
        err[want == 0] = np.abs(got[want == 0])
        assert err.max() < 4e-7, (name, float(err.max()), float(x32[err.argmax()]))
    assert utils.value_rescale(torch.zeros(1), eps).item() == 0.0
    # the reference's function is untouched: no eps x term, no cancellation-free form
    y = torch.tensor([0.5, -3.0])
    assert torch.equal(utils.invertical_vf(y), torch.sign(y) * (torch.sqrt(torch.abs(y) + 1) - 1))


# ------------------------------------------------------------------------------------------------ 3. drop-in Actor
def _actor(monkeypatch, tmp_path, **env):
    for k, v in dict(R2D2_OBS_SIZE="5", R2D2_N_ACTIONS="2", R2D2_HIDDEN="32", **env).items():
        monkeypatch.setenv(k, v)
    monkeypatch.chdir(tmp_path)
    import sys
    for m in ("actor", "utils"):
        sys.modules.pop(m, None)
    import actor as dropin_actor
    return dropin_actor.Actor(0)


@pytest.mark.parametrize("rescaling,metric", MODES)
def test_actor_calc_priorities_match_oracle(monkeypatch, tmp_path, rescaling, metric):
    env = {}
    if rescaling != "reference":
        env.update(R2D2_VALUE_RESCALING=rescaling, R2D2_RESCALING_EPS="0.01")
    if metric != "squared":
        env["R2D2_PRIORITY_METRIC"] = metric
    a = _actor(monkeypatch, tmp_path, **env)
    eps = 0.01 if rescaling == "invertible" else 1e-3
    assert (a.td_options.value_rescaling, a.td_options.priority_metric) == (rescaling, metric)
    torch.manual_seed(3)
    with torch.no_grad():                   # critic outputs of a few units, so that h_eps^-1 matters
        for net in (a.critic, a.target_critic):
            net.l3.weight.mul_(500.0)
            net.l3.bias.fill_(2.0)
    rng = np.random.default_rng(4)
    E, n = 75, a.n_step
    obs = rng.standard_normal((E + n, 5)).astype(np.float32)
    act = rng.uniform(-1, 1, (E + n, 2)).astype(np.float32)
    raw = (3 * rng.standard_normal(E + n)).astype(np.float32)
    term = np.zeros(E + n, np.float32)
    obs[E:], act[E:], raw[E:], term[E:] = 0, 0, 0, 1
    a.sequence = [(obs[i], act[i], [float(raw[i])], [float(term[i])]) for i in range(E + n)]
    a.calc_nstep_reward()
    a.calc_priorities()
    rew = np.asarray([row[2][0] for row in a.sequence])
    sd = lambda m: {k: v.numpy() for k, v in m.state_dict().items()}  # noqa: E731
    want = actor_oracle.episode_priorities(sd(a.critic), sd(a.target_actor), sd(a.target_critic), obs, act, rew, term,
                                 burn_in=a.burn_in_length, learning=a.learning_length, n_step=n, gamma=a.gamma,
                                 rescaling=rescaling, eps=eps, metric=metric)
    got = np.asarray(a.priority, np.float64)
    assert got.shape == want.shape == (E - 60,)
    assert rel_l2(got, want) < 1e-4, rel_l2(got, want)
    other = actor_oracle.episode_priorities(sd(a.critic), sd(a.target_actor), sd(a.target_critic), obs, act, rew, term,
                                  burn_in=a.burn_in_length, learning=a.learning_length, n_step=n, gamma=a.gamma,
                                  rescaling="reference" if rescaling == "invertible" else "invertible", eps=0.01,
                                  metric=metric)
    assert rel_l2(got, other) > 1e-2                 # the mode visibly matters on these inputs


# ------------------------------------------------------------------------------------------------ 4. validation
def test_td_options_environment():
    from r2d2_b200 import td_options as t
    assert t.from_environ({}) == t.TdOptions("reference", 1e-3, "squared")
    assert t.from_environ({}).is_default and t.from_environ({}).native() == (0, 1e-3, 0)
    o = t.from_environ({"R2D2_VALUE_RESCALING": "invertible", "R2D2_RESCALING_EPS": "0.01", "R2D2_PRIORITY_METRIC": "abs"})
    assert o == t.TdOptions("invertible", 0.01, "abs") and o.native() == (1, 0.01, 1) and not o.is_default
    for env, allowed in (({"R2D2_VALUE_RESCALING": "invertable"}, "reference, invertible"),
                         ({"R2D2_VALUE_RESCALING": "Invertible"}, "reference, invertible"),
                         ({"R2D2_PRIORITY_METRIC": "absolute"}, "squared, abs"),
                         ({"R2D2_PRIORITY_METRIC": ""}, "squared, abs"),
                         ({"R2D2_RESCALING_EPS": "1e-3x"}, "[0, 1]"), ({"R2D2_RESCALING_EPS": "nan"}, "[0, 1]"),
                         ({"R2D2_RESCALING_EPS": "-0.001"}, "[0, 1]"), ({"R2D2_RESCALING_EPS": "2"}, "[0, 1]"),
                         ({"R2D2_RESCALING_EPS": "inf"}, "[0, 1]")):
        with pytest.raises(ValueError) as e:
            t.from_environ(env)
        msg = str(e.value)
        assert next(iter(env)) in msg and allowed in msg, msg


def test_path_config_td_options_are_validated():
    from r2d2_b200 import engine
    cfg = engine.PathConfig(obs=3, act=1)
    assert (cfg.value_rescaling, cfg.rescaling_eps, cfg.priority_metric) == ("reference", 1e-3, "squared")
    engine.PathConfig(obs=3, act=1, value_rescaling="invertible", rescaling_eps=0.0, priority_metric="abs")
    engine.PathConfig(obs=3, act=1, value_rescaling="invertible", rescaling_eps=1.0)
    for bad in ({"value_rescaling": "h"}, {"value_rescaling": None}, {"priority_metric": "l1"},
                {"rescaling_eps": -1e-9}, {"rescaling_eps": 1.5}, {"rescaling_eps": float("nan")},
                {"rescaling_eps": float("inf")}, {"rescaling_eps": "0.001"}):
        with pytest.raises(ValueError):
            engine.PathConfig(obs=3, act=1, **bad)


def test_dropin_learner_reads_td_options(monkeypatch, tmp_path):
    c = fake_engine_learner(monkeypatch, tmp_path, R2D2_VALUE_RESCALING="invertible", R2D2_RESCALING_EPS="0.002",
                        R2D2_PRIORITY_METRIC="abs").engine.cfg
    assert (c.value_rescaling, c.rescaling_eps, c.priority_metric) == ("invertible", 0.002, "abs")
    for k in ("R2D2_VALUE_RESCALING", "R2D2_RESCALING_EPS", "R2D2_PRIORITY_METRIC"):
        monkeypatch.delenv(k)
    c = fake_engine_learner(monkeypatch, tmp_path).engine.cfg
    assert (c.value_rescaling, c.rescaling_eps, c.priority_metric) == ("reference", 1e-3, "squared")
    for bad in (dict(R2D2_VALUE_RESCALING="inverse"), dict(R2D2_PRIORITY_METRIC="l1"), dict(R2D2_RESCALING_EPS="-1")):
        with pytest.raises(ValueError):
            fake_engine_learner(monkeypatch, tmp_path, **bad)
        monkeypatch.delenv(next(iter(bad)))


def test_actor_pool_reads_td_options(monkeypatch, tmp_path):
    for k, v in dict(R2D2_OBS_SIZE="5", R2D2_N_ACTIONS="2", R2D2_HIDDEN="32", R2D2_VALUE_RESCALING="invertible",
                     R2D2_PRIORITY_METRIC="abs").items():
        monkeypatch.setenv(k, v)
    monkeypatch.chdir(tmp_path)
    from actor_pool import ActorPool, ModelsStepper
    pool = ActorPool([0], stepper=ModelsStepper(5, 2, 32, 1), priority_fn=lambda md, eps: ([], []))
    assert (pool.td_options.value_rescaling, pool.td_options.rescaling_eps, pool.td_options.priority_metric) == \
        ("invertible", 1e-3, "abs")
    monkeypatch.setenv("R2D2_PRIORITY_METRIC", "squre")
    with pytest.raises(ValueError, match="squared, abs"):
        ActorPool([0], stepper=ModelsStepper(5, 2, 32, 1), priority_fn=lambda md, eps: ([], []))


def test_checkpoint_options_mismatch_is_refused():
    """load_training_state compares the options before it touches any device memory."""
    from r2d2_b200 import engine
    eng = object.__new__(engine.LearnerEngine)
    for mine, saved in (
            (dict(value_rescaling="invertible"), {}),                                     # old checkpoint = reference
            (dict(priority_metric="abs"), {}),
            ({}, dict(value_rescaling="invertible", rescaling_eps=1e-3, priority_metric="squared")),
            (dict(value_rescaling="invertible", rescaling_eps=1e-3),
             dict(value_rescaling="invertible", rescaling_eps=1e-2, priority_metric="squared")),
            ({}, dict(value_rescaling="reference", rescaling_eps=1e-3, priority_metric="abs"))):
        eng.cfg = engine.PathConfig(obs=3, act=1, **mine)
        with pytest.raises(ValueError) as e:
            eng.load_training_state(dict(saved, actor={}, critic={}))
        msg = str(e.value)
        for o in (eng.td_options, saved):
            v = o.get("value_rescaling", "reference") if isinstance(o, dict) else o.value_rescaling
            assert repr(v) in msg, msg
        assert "saved with" in msg and "this engine runs" in msg


# ------------------------------------------------------------------------------------------------ 5. compiler report
TD_KERNELS = {"td_elem_kernel": 2, "td_reduce_kernel": 2, "td_priority_column_kernel": 4, "actor_priority_kernel": 4}


def _default_actor_kernel(name):
    """actor_priority_kernel<false, false> compiles to the SASS the kernel had before it became a template, which keeps
    its thread index in an 8-byte stack slot across the division slow-path calls of its window loop; a SASS diff against
    the earlier build pins that instantiation, so the checks here cover every other one."""
    return "actor_priority_kernelILb0ELb0E" in name


def test_td_kernels_do_not_spill():
    report, stderr = ptxas_report("elementwise.cu")
    found = {k: 0 for k in TD_KERNELS}
    for m in report:
        for k in TD_KERNELS:
            if k in m.group(1):
                found[k] += 1
                if not _default_actor_kernel(m.group(1)):
                    assert m.group(2) == m.group(3) == m.group(4) == "0", m.group(0)
    assert found == TD_KERNELS, stderr[-2000:]


def test_td_sass_has_every_instantiation_and_no_local_memory():
    sass = library_sass()
    for k, want in TD_KERNELS.items():
        funcs = functions(sass, k)
        flags = sorted("".join(re.findall(r"Lb([01])E", n)) for n in funcs)      # template flags, in order
        width = 1 if want == 2 else 2
        assert flags == ["".join(f) for f in itertools.product("01", repeat=width)], (k, sorted(funcs))
        for name, body in funcs.items():
            body_ops = [op for op, _ in ops(body)]
            if not _default_actor_kernel(name):
                assert not [op for op in body_ops if op.startswith(("LDL", "STL"))], f"local-memory traffic in {name}"

"""TD3's target on the host side: the oracle's Philox against Random123's known answers, the float64 oracle with the
twin against a torch-autograd float64 restatement on oracle/ref_port.py's nets (twin, smoothing, Polyak targets, joint
clipping), validation of PathConfig / the environment variables / checkpoints, and the compiler's report on the new
kernels (present, no spills, no local memory)."""
import copy

import numpy as np
import pytest
import torch

from conftest import rel_l2
from learner_harness import fake_engine_learner
from oracle import learner_oracle as lo
from oracle import ref_port
from oracle import target_noise as tn
from sass_report import functions, library_sass, ops, ptxas_report

SMALL = dict(obs=5, act=2, hidden=16, batch=4, burn_in=3, learning=5, n_step=2)


# ------------------------------------------------------------------------------------------------ 1. Philox
KAT = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
       ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
       ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
        (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]


@pytest.mark.parametrize("ctr,key,want", KAT)
def test_philox_known_answers(ctr, key, want):
    assert tuple(int(x) for x in tn.philox4x32_10(ctr, key)) == want


def test_noise_layout_and_range():
    """Four elements share one Philox block; u is an odd multiple of 2^-24 inside (0, 1); (seed, rank, iter) all key."""
    z = tn.normal(4096, 7, 0, 3)
    x = tn.philox4x32_10((np.uint64(1), np.uint64(3), np.uint64(0), np.uint64(0)), (np.uint64(7), np.uint64(0)))
    u = tn.unit_open(np.asarray(x))
    r01, r23 = np.sqrt(-2 * np.log(u[0])), np.sqrt(-2 * np.log(u[2]))
    assert np.allclose(z[4:8], [r01 * np.cos(2 * np.pi * u[1]), r01 * np.sin(2 * np.pi * u[1]),
                                r23 * np.cos(2 * np.pi * u[3]), r23 * np.sin(2 * np.pi * u[3])], rtol=0, atol=0)
    assert tn.unit_open(np.uint32(0)) == 2.0 ** -24 and tn.unit_open(np.uint32(0xffffffff)) == 1 - 2.0 ** -24
    for other in (tn.normal(4096, 8, 0, 3), tn.normal(4096, 7, 1, 3), tn.normal(4096, 7, 0, 4),
                  tn.normal(4096, 7, 0, 3 + 2 ** 32)):
        assert not np.any(other == z)
    a = tn.smooth(np.full(4096, 0.9), 1.0, 0.3, 7, 0, 3)
    low = 0.9 - 0.3                                    # the c clip binds below, the [-1, 1] clamp above
    assert a.max() == 1.0 and a.min() == low and np.any(a == low) and np.any((a > low) & (a < 1.0))


# ------------------------------------------------------------------------------------------------ 2. nets
def _port_params(seed=1, cfg=None):
    pc = ref_port.PathConfig(**(cfg or SMALL))
    port = ref_port.PortLearner(pc, seed=seed)
    sd = lambda m: {k: v.detach().numpy().astype(np.float64) for k, v in m.state_dict().items()}  # noqa: E731
    c2 = ref_port.PortCriticNet(pc.obs, pc.act, 0, pc.hidden)
    return pc, sd(port.actor), sd(port.critic), sd(c2)


# ------------------------------------------------------------------------------------------------ 3. vs autograd
def _autograd_run(pc, actor, critic, critic2, batches, *, sigma, clip_c, seed, tau, interval, max_norm):
    """TD3 in torch float64 autograd on the reference port's nets, row by row as the reference learner runs them."""
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        mk = lambda cls, sd: _load(cls(pc.obs, pc.act, 0, pc.hidden), sd)  # noqa: E731
        A, C1, C2 = (mk(ref_port.PortActorNet, actor), mk(ref_port.PortCriticNet, critic),
                     mk(ref_port.PortCriticNet, critic2))
        TA, TC1, TC2 = copy.deepcopy(A), copy.deepcopy(C1), copy.deepcopy(C2)
        opt_a = torch.optim.Adam(A.parameters(), lr=pc.actor_lr)
        critic_params = list(C1.parameters()) + list(C2.parameters())
        opt_c = torch.optim.Adam(critic_params, lr=pc.critic_lr)
        Bn, L, n = pc.burn_in, pc.learning, pc.n_step
        disc = pc.gamma ** n
        for it, batch in enumerate(batches):
            t = {k: torch.as_tensor(np.asarray(v, np.float64)) for k, v in batch.items()}
            obs, act = t["obs"], t["act"]
            rew, term = t["rew"].reshape(obs.shape[0], -1, 1), t["term"].reshape(obs.shape[0], -1, 1)
            with torch.no_grad():
                TA.set_state(t["ta_state"][0], t["ta_state"][1])
                a_next = torch.stack([TA(obs[k]) for k in range(Bn + n + L)][Bn + n:])
                if sigma > 0:
                    z = torch.as_tensor(tn.normal(a_next.numel(), seed, 0, it).reshape(a_next.shape))
                    a_next = torch.clamp(a_next + torch.clamp(sigma * z, -clip_c, clip_c), -1.0, 1.0)
                acts = torch.cat((act[:Bn + n], a_next), 0)
                TC1.set_state(t["tc_state"][0], t["tc_state"][1])
                TC2.reset_state()
                q1 = torch.stack([TC1(obs[k], acts[k]) for k in range(Bn + n + L)][Bn + n:])
                q2 = torch.stack([TC2(obs[k], acts[k]) for k in range(Bn + n + L)][Bn + n:])
                y = ref_port.value_rescale(rew[Bn:Bn + L] + disc * (1.0 - term[Bn + n - 1:Bn + n - 1 + L]) *
                                           torch.minimum(q1, q2))
            C1.set_state(t["c_state"][0], t["c_state"][1])
            C2.reset_state()
            qa = torch.stack([C1(obs[k], act[k]) for k in range(Bn + L)][Bn:])
            qb = torch.stack([C2(obs[k], act[k]) for k in range(Bn + L)][Bn:])
            opt_c.zero_grad()
            (torch.mean((qa - y) ** 2) + torch.mean((qb - y) ** 2)).backward()
            if max_norm > 0:
                torch.nn.utils.clip_grad_norm_(critic_params, max_norm)
            opt_c.step()
            A.reset_state()
            C1.reset_state()
            neg = []
            for i in range(L):
                A(obs[Bn + i])
                neg.append(-C1(obs[Bn + i], A(obs[Bn + i])))
            opt_a.zero_grad()
            torch.stack(neg).mean().backward()
            if max_norm > 0:
                torch.nn.utils.clip_grad_norm_(A.parameters(), max_norm)
            opt_a.step()
            for net in (A, C1, C2, TA, TC1, TC2):
                net.reset_state()
            if (it + 1) % interval == 0:
                with torch.no_grad():
                    for tgt, src in ((TA, A), (TC1, C1), (TC2, C2)):
                        for pt, ps in zip(tgt.parameters(), src.parameters()):
                            pt.copy_(pt * (1.0 - tau) + ps * tau)
        sd = lambda m: {k: v.detach().numpy().copy() for k, v in m.state_dict().items()}  # noqa: E731
        return {"actor": sd(A), "critic": sd(C1), "critic2": sd(C2), "target_actor": sd(TA), "target_critic": sd(TC1),
                "target_critic2": sd(TC2), "m_critic2": [opt_c.state[p]["exp_avg"].numpy() for p in C2.parameters()]}
    finally:
        torch.set_default_dtype(old)


def _load(net, sd):
    net.load_state_dict({k: torch.as_tensor(v) for k, v in sd.items()})
    return net


@pytest.mark.parametrize("sigma,clip_c", [(0.2, 0.5), (1.5, 0.3)])
def test_oracle_matches_torch_autograd(sigma, clip_c):
    pc, a, c, c2 = _port_params(seed=4)
    batches = [ref_port.synthetic_batch(pc, seed=10 + i) for i in range(4)]
    probe = lo.OracleLearner(a, c, critic2=c2, twin=True, burn_in=pc.burn_in, learning=pc.learning, n_step=pc.n_step,
                             grad_clip=1e30)
    probe.iteration(batches[0])
    max_norm = 0.1 * min(probe.norms.values())             # both clip from the first iteration on
    ol = lo.OracleLearner(a, c, critic2=c2, twin=True, target_noise=sigma, target_noise_clip=clip_c, target_noise_seed=3,
                          target_tau=0.05, grad_clip=max_norm, burn_in=pc.burn_in, learning=pc.learning,
                          n_step=pc.n_step, target_interval=1)
    for b in batches:
        ol.iteration(b)
    want = _autograd_run(pc, a, c, c2, batches, sigma=sigma, clip_c=clip_c, seed=3, tau=0.05, interval=1,
                         max_norm=max_norm)
    errs = {f"{net}/{k}": rel_l2(getattr(ol, net)[k], want[net][k])
            for net in ("actor", "critic", "critic2", "target_actor", "target_critic", "target_critic2")
            for k in lo.PARAM_KEYS}
    for i, k in enumerate(lo.PARAM_KEYS):
        errs[f"m/critic2/{k}"] = rel_l2(ol.critic2_adam["m/" + k], want["m_critic2"][i])
    assert max(errs.values()) < 1e-10, {k: v for k, v in errs.items() if v >= 1e-10}
    # the options visibly matter: the same run without the twin's minimum or without noise ends elsewhere
    plain = lo.OracleLearner(a, c, critic2=c2, twin=True, target_tau=0.05, grad_clip=max_norm, burn_in=pc.burn_in,
                             learning=pc.learning, n_step=pc.n_step, target_interval=1)
    for b in batches:
        plain.iteration(b)
    assert rel_l2(plain.critic["l3.weight"], ol.critic["l3.weight"]) > 1e-6


# ------------------------------------------------------------------------------------------------ 4. validation
def test_path_config_td3_fields_are_validated():
    from r2d2_b200 import engine
    cfg = engine.PathConfig(obs=3, act=1)
    assert (cfg.twin_critic, cfg.target_noise, cfg.target_noise_clip, cfg.target_noise_seed) == (False, 0.0, 0.5, 0)
    engine.PathConfig(obs=3, act=1, twin_critic=True, target_noise=0.2, target_noise_clip=0.5, target_noise_seed=2 ** 32 - 1)
    engine.PathConfig(obs=3, act=1, target_noise=np.float32(0.2))
    for bad in ({"twin_critic": 1}, {"twin_critic": "yes"}, {"target_noise": -0.1}, {"target_noise": float("nan")},
                {"target_noise": float("inf")}, {"target_noise": "0.2"}, {"target_noise_clip": 0.0},
                {"target_noise_clip": -1.0}, {"target_noise_clip": float("inf")}, {"target_noise_seed": -1},
                {"target_noise_seed": 2 ** 32}, {"target_noise_seed": 1.5}, {"target_noise_seed": True}):
        with pytest.raises(ValueError):
            engine.PathConfig(obs=3, act=1, **bad)


def test_td3_environment():
    from r2d2_b200 import td3_options as o
    assert o.from_environ({}) == dict(twin_critic=False, target_noise=0.0, target_noise_clip=0.5, target_noise_seed=0)
    assert o.from_environ({"R2D2_TWIN_CRITIC": "1", "R2D2_TARGET_NOISE": "0.2", "R2D2_TARGET_NOISE_CLIP": "0.4",
                           "R2D2_TARGET_NOISE_SEED": "9"}) == \
        dict(twin_critic=True, target_noise=0.2, target_noise_clip=0.4, target_noise_seed=9)
    for env, allowed in (({"R2D2_TWIN_CRITIC": "true"}, "0, 1"), ({"R2D2_TWIN_CRITIC": ""}, "0, 1"),
                         ({"R2D2_TARGET_NOISE": "-0.1"}, ">= 0"), ({"R2D2_TARGET_NOISE": "nan"}, ">= 0"),
                         ({"R2D2_TARGET_NOISE": "x"}, ">= 0"), ({"R2D2_TARGET_NOISE_CLIP": "0"}, "> 0"),
                         ({"R2D2_TARGET_NOISE_CLIP": "inf"}, "> 0"), ({"R2D2_TARGET_NOISE_SEED": "-1"}, "[0, 2**32)"),
                         ({"R2D2_TARGET_NOISE_SEED": "1.5"}, "[0, 2**32)")):
        with pytest.raises(ValueError) as e:
            o.from_environ(env)
        msg = str(e.value)
        assert next(iter(env)) in msg and allowed in msg, msg


def test_dropin_learner_reads_td3_options(monkeypatch, tmp_path):
    c = fake_engine_learner(monkeypatch, tmp_path, R2D2_TWIN_CRITIC="1", R2D2_TARGET_NOISE="0.2",
                        R2D2_TARGET_NOISE_CLIP="0.5", R2D2_TARGET_NOISE_SEED="4").engine.cfg
    assert (c.twin_critic, c.target_noise, c.target_noise_clip, c.target_noise_seed) == (True, 0.2, 0.5, 4)
    for k in ("R2D2_TWIN_CRITIC", "R2D2_TARGET_NOISE", "R2D2_TARGET_NOISE_CLIP", "R2D2_TARGET_NOISE_SEED"):
        monkeypatch.delenv(k)
    c = fake_engine_learner(monkeypatch, tmp_path).engine.cfg
    assert (c.twin_critic, c.target_noise) == (False, 0.0)
    with pytest.raises(ValueError, match="0, 1"):
        fake_engine_learner(monkeypatch, tmp_path, R2D2_TWIN_CRITIC="2")


def test_checkpoint_twin_mismatch_is_refused():
    """load_training_state compares the twin setting before it touches any device memory; no key = single critic."""
    from r2d2_b200 import engine
    eng = object.__new__(engine.LearnerEngine)
    for mine, saved in ((dict(twin_critic=True), {}), (dict(twin_critic=True), dict(twin_critic=False)),
                        ({}, dict(twin_critic=True))):
        eng.cfg = engine.PathConfig(obs=3, act=1, **mine)
        with pytest.raises(ValueError, match="twin_critic"):
            eng.load_training_state(dict(saved, actor={}, critic={}))


# ------------------------------------------------------------------------------------------------ 5. compiler report
TD3_KERNELS = ("target_smoothing_kernel", "q_min_kernel")


def test_td3_kernels_do_not_spill():
    report, stderr = ptxas_report("td3.cu")
    found = dict.fromkeys(TD3_KERNELS, 0)
    for m in report:
        for k in TD3_KERNELS:
            if k in m.group(1):
                found[k] += 1
                assert m.group(2) == m.group(3) == m.group(4) == "0", m.group(0)
    assert found == dict.fromkeys(TD3_KERNELS, 1), stderr[-2000:]


def test_td3_sass_present_without_local_memory():
    sass = library_sass()
    for k in TD3_KERNELS:
        funcs = functions(sass, k)
        assert len(funcs) == 1, (k, sorted(funcs))
        for name, body in funcs.items():
            body_ops = [op for op, _ in ops(body)]
            assert not [op for op in body_ops if op.startswith(("LDL", "STL"))], f"local-memory traffic in {name}"
            if k == "target_smoothing_kernel":   # the precise functions, not the fast-math approximations alone
                assert "IMAD.HI.U32" in body_ops or any(op.startswith("IMAD.WIDE.U32") for op in body_ops), name

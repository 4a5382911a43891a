"""r2d2_policy_step and ActorPool on the GPU: the step kernels against the float64 policy step of
oracle/actor_oracle, lane independence bit for bit, shape errors, and
the pool end to end (files the drop-in nets reproduce, priorities against oracle/actor_oracle, model.pt reload, and a
learner that ingests the files)."""
import os
import shutil
import types

import numpy as np
import pytest
import torch

from conftest import rel_l2
from oracle import actor_oracle
from oracle.actor_oracle import NETS, policy_params

pytestmark = pytest.mark.gpu

CASES = [(O, A, H, N) for (O, A, H) in ((24, 6, 128), (17, 6, 256), (376, 17, 512), (5, 1, 32))
         for N in (1, 3, 64, 256) if N < 256 or H <= 256]


@pytest.mark.parametrize("O,A,H,N", CASES)
def test_policy_step_matches_float64_oracle(O, A, H, N):
    from r2d2_b200.policy_step import PolicyStepper
    md = policy_params(O, A, H, seed=O + H + N)
    st = PolicyStepper(O, A, H, N, device="cuda", max_episode_steps=64)
    st.load(md)
    P = {n: {k: v.astype(np.float64) for k, v in md[n].items()} for n in NETS}
    rng = np.random.default_rng(N)
    ref = np.zeros((4, 2, N, H))
    st.reset(range(N))
    for s in range(200):
        lanes = [n for n in range(N) if s > 0 and s % 50 == (7 * n) % 50]   # staggered episode starts
        if lanes:
            st.reset(lanes)
            ref[:, :, lanes] = 0
        obs = rng.standard_normal((N, O)).astype(np.float32)
        mu = st.step(obs)
        mu_ref, ref = actor_oracle.policy_step(P, obs.astype(np.float64), ref)
        got = st.current_states().cpu().numpy()
        errs = {"mu": rel_l2(mu, mu_ref)}
        for k, name in enumerate(NETS):
            errs[name + ".h"] = rel_l2(got[k, 0], ref[k, 0])
            errs[name + ".c"] = rel_l2(got[k, 1], ref[k, 1])
        assert max(errs.values()) < 2e-5, (s, errs)


ACT = 6


def _raw_step(params, obs, state_in):
    from r2d2_b200.policy_step import policy_step
    mu = torch.empty((obs.shape[0], ACT), device="cuda")
    out = torch.empty_like(state_in)
    policy_step(params, obs, state_in, out, mu)
    return mu, out


def test_lanes_are_bitwise_independent():
    from r2d2_b200.policy_step import PolicyStepper
    O, H, N = 17, 256, 64
    st = PolicyStepper(O, ACT, H, 1, device="cuda")
    st.load(policy_params(O, ACT, H, seed=5))
    g = torch.Generator(device="cuda").manual_seed(0)
    obs = torch.randn((N, O), device="cuda", generator=g)
    s_in = 0.5 * torch.randn((4, 2, N, H), device="cuda", generator=g)
    mu, out = _raw_step(st.params, obs, s_in)
    mu2, out2 = _raw_step(st.params, obs, s_in)
    assert torch.equal(mu, mu2) and torch.equal(out, out2), "two runs differ"
    for n in range(N):
        m1, o1 = _raw_step(st.params, obs[n:n + 1].contiguous(), s_in[:, :, n:n + 1].contiguous())
        assert torch.equal(m1[0], mu[n]) and torch.equal(o1[:, :, 0], out[:, :, n]), f"lane {n} depends on N"


@pytest.mark.parametrize("O,A,H,N", [(5, 2, 64, 0), (5, 2, 64, 257), (5, 2, 48, 4), (5, 65, 64, 4)])
def test_unsupported_shapes_raise(O, A, H, N):
    from ctypes import c_void_p
    from r2d2_b200 import native as nv
    buf = torch.zeros(1 << 22, device="cuda")
    p = nv.dptr(buf)
    ptrs = (c_void_p * 4)(p.value, p.value, p.value, p.value)
    rc = nv.lib().r2d2_policy_step(nv.byref(nv.NetShape(O, A, H, 0)), ptrs, p, p, nv.dptr(buf[1 << 21:]), p, N, p,
                                   nv.current_stream())
    assert rc == -3
    with pytest.raises(nv.NativeError, match="unsupported shape"):
        nv.check(rc)


# ------------------------------------------------------------------------------------------------ ActorPool
O_P, A_P, H_P, LANES = 5, 2, 64, 8


@pytest.fixture(scope="module")
def pool_run(tmp_path_factory):
    d = tmp_path_factory.mktemp("pool")
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("R2D2_OBS_SIZE", str(O_P))
        mp.setenv("R2D2_N_ACTIONS", str(A_P))
        mp.setenv("R2D2_HIDDEN", str(H_P))
        mp.chdir(d)
        os.makedirs("memory_data")
        os.makedirs("model_data")
        from actor_pool import ActorPool, initial_model_dict
        torch.manual_seed(0)
        md = initial_model_dict(O_P, A_P, H_P)
        for sd in md.values():
            sd["l3.weight"].uniform_(-0.3, 0.3)                 # Q values well above the rounding of tiny TD errors
        torch.save(md, "model_data/model.pt")                  # the pool starts from the learner's weights
        pool = ActorPool(range(LANES), device="cuda", noise_std=0.0)
        assert torch.equal(pool.model_dict["critic"]["l3.weight"], md["critic"]["l3.weight"])
        seen = []
        gpu_prio = pool.priority_fn

        def prio(model_dict, episodes):
            out = gpu_prio(model_dict, episodes)
            seen.append((model_dict, episodes, out))
            return out
        pool.priority_fn = prio
        for i, env in enumerate(pool.envs):
            env.episode_len = 66 + 12 * i                       # 66 .. 150
        pool.run(max_steps=605)                                 # every lane has saved 4 episodes
        files = {i: torch.load(f"memory_data/memory{i}.pt", weights_only=False) for i in range(LANES)}
        yield types.SimpleNamespace(dir=d, pool=pool, seen=seen, files=files)


def _cpu_nets(model_dict):
    from models import ActorNet, CriticNet
    nets = [cls(O_P, A_P, 0, hidden=H_P).eval() for cls in (ActorNet, ActorNet, CriticNet, CriticNet)]
    for net, name in zip(nets, NETS):
        net.load_state_dict(model_dict[name])
    return nets


@torch.no_grad()
def _teacher_step(nets, state, obs):
    for k, net in enumerate(nets):
        net.set_state(torch.as_tensor(state[k, 0])[None], torch.as_tensor(state[k, 1])[None])
    x = torch.as_tensor(obs)[None]
    mu = nets[0](x)
    nets[2](x, mu)
    nets[3](x, nets[1](x))
    return mu[0].numpy(), np.stack([np.stack([n.hx[0].numpy(), n.cx[0].numpy()]) for n in nets])


def test_pool_files_follow_the_dropin_nets(pool_run):
    from replay_memory import pack_episode
    nets = _cpu_nets(pool_run.pool.model_dict)
    for i, payload in pool_run.files.items():
        assert len(payload["replay_memory"]) == 4
        E = 66 + 12 * i
        for rows, states, prio in zip(payload["replay_memory"], payload["recurrent_state"], payload["priority"]):
            obs, act, rew, term, st = pack_episode(rows, states, hidden=H_P)
            assert obs.shape[0] == E + 5 and st.shape[0] == E and len(prio) == E - 60
            assert not st[0].any()
            for e in range(E):
                mu, nxt = _teacher_step(nets, st[e], obs[e])
                np.testing.assert_allclose(act[e], np.clip(mu, -1, 1), atol=1e-4)
                if e + 1 < E:
                    np.testing.assert_allclose(nxt, st[e + 1], atol=1e-4)


def test_pool_priorities_match_actor_oracle(pool_run):
    n = 0
    for model_dict, episodes, (prios, rews) in pool_run.seen:
        for (obs, act, raw, term), p, r in zip(episodes, prios, rews):
            want_r = actor_oracle.nstep_rewards(raw, 5, 0.997)
            want_p = actor_oracle.episode_priorities(model_dict["critic"], model_dict["target_actor"],
                                                     model_dict["target_critic"], obs, act, want_r, term,
                                                     burn_in=20, learning=40, n_step=5, gamma=0.997)
            assert rel_l2(r, want_r) < 1e-3 and rel_l2(p, want_p) < 1e-3
            n += 1
    assert n >= 4 * LANES
    # the files carry those n-step rewards
    by_obs = {ep[0].tobytes(): r for _, episodes, (_, rews) in pool_run.seen for ep, r in zip(episodes, rews)}
    for payload in pool_run.files.values():
        for rows in payload["replay_memory"]:
            want = by_obs[np.stack([r[0] for r in rows]).astype(np.float32).tobytes()]
            np.testing.assert_array_equal(np.float32([r[2][0] for r in rows]), want)


def test_learner_ingests_pool_files(pool_run, monkeypatch, tmp_path):
    monkeypatch.setenv("R2D2_OBS_SIZE", str(O_P))
    monkeypatch.setenv("R2D2_N_ACTIONS", str(A_P))
    monkeypatch.setenv("R2D2_HIDDEN", str(H_P))
    monkeypatch.setenv("R2D2_BATCH", "4")
    monkeypatch.chdir(tmp_path)
    os.makedirs("model_data")
    shutil.copytree(os.path.join(pool_run.dir, "memory_data"), "memory_data")
    import learner
    lr = learner.Learner(n_actors=LANES)
    lr.model_save_interval = 2
    lr.memory_update_interval = 2
    lr.run(max_steps=4)
    assert lr.engine.step_count == 4
    assert lr.memory.sequence_counter >= 400 and len(lr.memory.memory) == 4 * LANES
    assert not [f for f in os.listdir("memory_data") if f.endswith(".pt")], "every pool file was ingested"


def test_pool_follows_new_model_pt(pool_run):
    pool = pool_run.pool
    cwd = os.getcwd()
    os.chdir(pool_run.dir)
    try:
        from actor_pool import initial_model_dict
        torch.manual_seed(123)
        new = initial_model_dict(O_P, A_P, H_P)
        for sd in new.values():
            sd["l3.weight"].uniform_(-0.3, 0.3)                 # a head that moves mu visibly
        torch.save(new, "model_data/model.pt")
        pool.run(max_steps=500 - pool.steps % 500)              # the reload happens on the 500th step
        assert pool.model_dict is not None and torch.equal(pool.model_dict["actor"]["l3.weight"], new["actor"]["l3.weight"])
        state = pool.stepper.current_states().cpu().numpy()
        obs = pool.obs.copy()
        pool.step()
        nets = _cpu_nets(new)
        for lane in range(LANES):
            mu, _ = _teacher_step(nets, state[:, :, lane], obs[lane])
            np.testing.assert_allclose(pool.last_mu[lane], mu, atol=1e-4)
        old_nets = _cpu_nets(pool_run.seen[0][0])
        mu_old, _ = _teacher_step(old_nets, state[:, :, 0], obs[0])
        assert np.abs(mu_old - pool.last_mu[0]).max() > 1e-3
    finally:
        os.chdir(cwd)

"""ActorPool host bookkeeping on the CPU: the models.py nets stepped by ModelsStepper and the float64 actor oracle for
priorities stand in for the GPU pieces.  The files it writes must be what Actor.run writes."""
import os

import numpy as np
import pytest
import torch

from oracle import actor_oracle

N_STEP, GAMMA, BURN_IN, LEARNING = 5, 0.997, 20, 40


def _oracle_priorities(model_dict, episodes):
    prios, rews = [], []
    for obs, act, raw, term in episodes:
        rew = actor_oracle.nstep_rewards(raw, N_STEP, GAMMA)
        prios.append(actor_oracle.episode_priorities(
            *(model_dict[k] for k in ("critic", "target_actor", "target_critic")), obs, act, rew, term,
            burn_in=BURN_IN, learning=LEARNING, n_step=N_STEP, gamma=GAMMA).astype(np.float32))
        rews.append(rew.astype(np.float32))
    return prios, rews


@pytest.fixture
def pool_env(monkeypatch, tmp_path):
    monkeypatch.setenv("R2D2_OBS_SIZE", "5")
    monkeypatch.setenv("R2D2_N_ACTIONS", "2")
    monkeypatch.setenv("R2D2_HIDDEN", "32")
    monkeypatch.chdir(tmp_path)
    os.makedirs("memory_data")
    os.makedirs("model_data")
    return tmp_path


def test_pool_files_match_actor_format(pool_env):
    from actor_pool import ActorPool, ModelsStepper
    from replay_memory import pack_episode
    torch.manual_seed(0)
    # max_episode_steps 80 < 4 episodes of 70 steps: the state ring wraps
    stepper = ModelsStepper(5, 2, 32, 3, max_episode_steps=80)
    pool = ActorPool([3, 7, 9], stepper=stepper, priority_fn=_oracle_priorities, seed=1)
    for env, n in zip(pool.envs, (70, 65, 50)):       # lane 2's episodes are shorter than 60 steps: all dropped
        env.episode_len = n
    pool.run(max_steps=285)
    assert sorted(os.listdir("memory_data")) == ["memory3.pt", "memory7.pt"]
    nets = [m.eval() for m in stepper.nets]
    for aid, E in ((3, 70), (7, 65)):
        payload = torch.load(f"memory_data/memory{aid}.pt", weights_only=False)
        assert len(payload["replay_memory"]) == 4
        for rows, states, prio, total in zip(payload["replay_memory"], payload["recurrent_state"],
                                             payload["priority"], payload["total_priority"]):
            obs, act, rew, term, st = pack_episode(rows, states, hidden=32)
            assert obs.shape == (E + N_STEP, 5) and act.shape == (E + N_STEP, 2)
            assert st.shape == (E, 4, 2, 32)
            assert len(prio) == E - BURN_IN - LEARNING
            assert np.all(np.isfinite(prio)) and abs(total - sum(prio)) < 1e-3
            assert not st[0].any(), "an episode starts from the zero state"
            assert term[E - 1] == 1 and not term[:E - 1].any() and term[E:].all()
            assert not obs[E:].any() and not rew[E:].any()
            # teacher forcing through the same nets: state e + 1 follows from state e and obs e
            with torch.no_grad():
                for e in range(E - 1):
                    for k, net in enumerate(nets):
                        net.set_state(torch.from_numpy(st[e, k, 0][None]), torch.from_numpy(st[e, k, 1][None]))
                    x = torch.from_numpy(obs[e][None])
                    mu = nets[0](x)
                    nets[2](x, mu)
                    nets[3](x, nets[1](x))
                    for k, net in enumerate(nets):
                        np.testing.assert_allclose(net.hx[0].numpy(), st[e + 1, k, 0], atol=1e-6)
                        np.testing.assert_allclose(net.cx[0].numpy(), st[e + 1, k, 1], atol=1e-6)
                    assert np.all(np.abs(act[e]) <= 1)


def test_pool_rewards_are_nstep_sums(pool_env):
    from actor_pool import ActorPool, ModelsStepper
    torch.manual_seed(0)
    seen = []

    def prio(model_dict, episodes):
        seen.extend(episodes)
        return _oracle_priorities(model_dict, episodes)
    pool = ActorPool([0], stepper=ModelsStepper(5, 2, 32, 1), priority_fn=prio, noise_std=0.0)
    pool.envs[0].episode_len = 62
    pool.run(max_steps=62)
    assert len(seen) == 1 and len(pool.memories[0].memory) == 1
    rows = pool.memories[0].memory[0]
    obs, act, raw, term = seen[0]
    assert raw.shape == (62 + N_STEP,) and not raw[62:].any()
    np.testing.assert_allclose([r[2][0] for r in rows], actor_oracle.nstep_rewards(raw, N_STEP, GAMMA), rtol=1e-6)
    np.testing.assert_array_equal(np.stack([r[1] for r in rows]), act)


def test_ring_overflow_names_max_episode_steps():
    from actor_pool import ModelsStepper
    st = ModelsStepper(3, 1, 32, 2, max_episode_steps=10)
    st.reset([0, 1])
    obs = np.zeros((2, 3), np.float32)
    for _ in range(10):
        st.step(obs)
    with pytest.raises(RuntimeError, match="max_episode_steps"):
        st.step(obs)
    st.reset([0, 1])
    st.step(obs)
    assert st.episode_states(0, st.t - 1, st.t).shape == (1, 4, 2, 32)

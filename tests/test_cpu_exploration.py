"""Actor exploration on the host: the R2D2_EXPLORATION* options and their refusals, the log-spaced sigma schedule, the
product's numpy Philox and noise against the oracle's, the OU recurrence against float64, the drop-in Actor against a
one-lane ActorPool on the CPU (same episodes bit for bit), the reference mode's unchanged noise sources, and the
compiler's report on the new head kernel."""
import os

import numpy as np
import pytest
import torch

import exploration_oracle as xo
from oracle import target_noise as tn
from sass_report import functions, library_sass, ops, ptxas_report
from test_cpu_td3 import KAT


def _ex():
    from r2d2_b200 import exploration
    return exploration


# ------------------------------------------------------------------------------------------------ 1. options
def test_defaults_are_the_reference():
    ex = _ex()
    o = ex.from_environ({})
    assert o == ex.Exploration() and o.mode == "reference"
    assert ex.from_environ({"R2D2_EXPLORATION": "reference"}) == o


def test_environment_values():
    ex = _ex()
    o = ex.from_environ({"R2D2_EXPLORATION": "ou", "R2D2_EXPLORATION_SIGMA": "0.4", "R2D2_EXPLORATION_SIGMA_MIN": "0.05",
                         "R2D2_EXPLORATION_ACTORS": "16", "R2D2_EXPLORATION_OU_THETA": "0.2",
                         "R2D2_EXPLORATION_SEED": "4294967295"})
    assert (o.mode, o.sigma, o.sigma_min, o.actors, o.theta, o.seed) == ("ou", 0.4, 0.05, 16, 0.2, 2 ** 32 - 1)
    assert o.kind == 1 and ex.from_environ({"R2D2_EXPLORATION": "gaussian"}).kind == 0
    assert o.one_minus_theta == np.float32(0.8)
    g = ex.from_environ({"R2D2_EXPLORATION": "gaussian", "R2D2_EXPLORATION_SIGMA": "0"})
    assert g.sigma == 0.0 and np.all(g.sigmas(range(5)) == 0)


@pytest.mark.parametrize("env,allowed", [
    ({"R2D2_EXPLORATION": "normal"}, "reference, gaussian, ou"),
    ({"R2D2_EXPLORATION": ""}, "reference, gaussian, ou"),
    ({"R2D2_EXPLORATION": "gaussian", "R2D2_EXPLORATION_SIGMA": "-0.1"}, ">= 0"),
    ({"R2D2_EXPLORATION": "gaussian", "R2D2_EXPLORATION_SIGMA": "nan"}, ">= 0"),
    ({"R2D2_EXPLORATION": "gaussian", "R2D2_EXPLORATION_SIGMA": "inf"}, ">= 0"),
    ({"R2D2_EXPLORATION": "gaussian", "R2D2_EXPLORATION_SIGMA": "x"}, ">= 0"),
    ({"R2D2_EXPLORATION": "gaussian", "R2D2_EXPLORATION_ACTORS": "4", "R2D2_EXPLORATION_SIGMA_MIN": "0.5"}, "(0, "),
    ({"R2D2_EXPLORATION": "gaussian", "R2D2_EXPLORATION_ACTORS": "4", "R2D2_EXPLORATION_SIGMA_MIN": "0"}, "(0, "),
    ({"R2D2_EXPLORATION": "gaussian", "R2D2_EXPLORATION_ACTORS": "4", "R2D2_EXPLORATION_SIGMA_MIN": "-1"}, "(0, "),
    ({"R2D2_EXPLORATION": "gaussian", "R2D2_EXPLORATION_ACTORS": "0"}, "integers >= 1"),
    ({"R2D2_EXPLORATION": "gaussian", "R2D2_EXPLORATION_ACTORS": "2.5"}, "integers >= 1"),
    ({"R2D2_EXPLORATION": "ou", "R2D2_EXPLORATION_OU_THETA": "0"}, "(0, 1]"),
    ({"R2D2_EXPLORATION": "ou", "R2D2_EXPLORATION_OU_THETA": "1.5"}, "(0, 1]"),
    ({"R2D2_EXPLORATION": "ou", "R2D2_EXPLORATION_OU_THETA": "nan"}, "(0, 1]"),
    ({"R2D2_EXPLORATION": "gaussian", "R2D2_EXPLORATION_OU_THETA": "0.15"}, "ou only"),
    ({"R2D2_EXPLORATION": "ou", "R2D2_EXPLORATION_SEED": "-1"}, "[0, 2**32)"),
    ({"R2D2_EXPLORATION": "ou", "R2D2_EXPLORATION_SEED": str(2 ** 32)}, "[0, 2**32)"),
    ({"R2D2_EXPLORATION": "ou", "R2D2_EXPLORATION_SEED": "1.5"}, "[0, 2**32)"),
])
def test_malformed_values_raise_and_name_the_allowed_ones(env, allowed):
    with pytest.raises(ValueError) as e:
        _ex().from_environ(env)
    msg = str(e.value)
    assert allowed in msg and list(env)[-1] in msg, msg


@pytest.mark.parametrize("name", ["R2D2_EXPLORATION_SIGMA", "R2D2_EXPLORATION_SIGMA_MIN", "R2D2_EXPLORATION_ACTORS",
                                  "R2D2_EXPLORATION_OU_THETA", "R2D2_EXPLORATION_SEED"])
@pytest.mark.parametrize("mode", [None, "reference"])
def test_other_variables_under_reference_raise(name, mode):
    env = {name: "0.3" if "ACTORS" not in name and "SEED" not in name else "3"}
    if mode:
        env["R2D2_EXPLORATION"] = mode
    with pytest.raises(ValueError, match=name):
        _ex().from_environ(env)


def test_sigma_min_without_actors_raises():
    ex = _ex()
    with pytest.raises(ValueError, match="R2D2_EXPLORATION_ACTORS"):
        ex.from_environ({"R2D2_EXPLORATION": "gaussian", "R2D2_EXPLORATION_SIGMA_MIN": "0.1"})
    with pytest.raises(ValueError, match="number of actors"):
        ex.Exploration("gaussian", 0.3, 0.1)
    # sigma_min equal to sigma needs no N
    assert ex.from_environ({"R2D2_EXPLORATION": "gaussian", "R2D2_EXPLORATION_SIGMA_MIN": "0.3"}).actors is None


def test_actor_id_beyond_the_schedule_raises():
    ex = _ex()
    o = ex.Exploration("gaussian", 0.4, 0.05, 16)
    o.sigmas(range(16))
    with pytest.raises(ValueError, match="actor id 16 >= R2D2_EXPLORATION_ACTORS=16"):
        o.sigmas([3, 16])
    with pytest.raises(ValueError, match="actor id 4"):                # N without a spread still bounds the ids
        ex.Exploration("gaussian", 0.3, None, 4).sigmas([4])
    with pytest.raises(ValueError, match="actor id"):
        ex.HostNoise(o, [20], 3)


def test_direct_construction_is_validated():
    ex = _ex()
    for bad in (dict(mode="x"), dict(sigma=-1.0), dict(sigma=float("nan")), dict(sigma_min=0.5, actors=3),
                dict(actors=0), dict(actors=True), dict(theta=0.0), dict(theta=1.01), dict(seed=-1), dict(seed=2 ** 32),
                dict(seed=1.0)):
        with pytest.raises(ValueError):
            ex.Exploration(**dict(dict(mode="ou"), **bad))


# ------------------------------------------------------------------------------------------------ 2. schedule
@pytest.mark.parametrize("smax,smin,n", [(0.4, 0.05, 16), (0.3, 0.01, 256), (1.0, 0.999, 3), (0.7, 0.1, 2)])
def test_schedule(smax, smin, n):
    o = _ex().Exploration("gaussian", smax, smin, n)
    s = o.sigmas(range(n))
    assert s.dtype == np.float32
    assert s[0] == np.float32(smax) and s[-1] == np.float32(smin)
    assert np.all(np.diff(s.astype(np.float64)) <= 0) and s[0] > s[-1]
    i = np.arange(n, dtype=np.float64)
    want = (smax * (smin / smax) ** (i / (n - 1))).astype(np.float32)     # float64, rounded to float32 once
    want[-1] = np.float32(smin)
    assert np.array_equal(s, want)
    assert np.array_equal(o.sigmas([n - 1, 0]), s[[n - 1, 0]])          # by id, not by position


def test_schedule_of_one_actor_is_sigma_max():
    ex = _ex()
    assert np.array_equal(ex.Exploration("gaussian", 0.4, 0.05, 1).sigmas([0]), np.float32([0.4]))
    assert np.array_equal(ex.Exploration("gaussian", 0.4).sigmas([0, 5, 900]), np.full(3, 0.4, np.float32))


# ------------------------------------------------------------------------------------------------ 3. generator
@pytest.mark.parametrize("ctr,key,want", KAT)
def test_product_philox_known_answers(ctr, key, want):
    assert tuple(int(x) for x in _ex().philox4x32_10(ctr, key)) == want


def test_product_philox_matches_oracle():
    rng = np.random.default_rng(0)
    ctr = [rng.integers(0, 2 ** 32, 4096, dtype=np.uint64) for _ in range(4)]
    key = [rng.integers(0, 2 ** 32, 4096, dtype=np.uint64) for _ in range(2)]
    for a, b in zip(_ex().philox4x32_10(ctr, key), tn.philox4x32_10(ctr, key)):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("step", [0, 7, 2 ** 32 + 5])
def test_product_noise_matches_float64(step):
    """The host z is the fp32 restatement of the kernel's: within 2 ulp of the float64 value (logf and sincospif are
    taken correctly rounded here; the kernel's are within 1 ulp of that)."""
    ids, A = [0, 1, 5, 255, 70000], 17
    z = _ex().normal(ids, step, A, 9)
    want = xo.normal(ids, step, A, 9)
    assert z.dtype == np.float32
    ulp = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
    assert np.all(np.abs(z - want) <= 2 * ulp), np.max(np.abs(z - want) / ulp)
    # each key and counter word matters, and c3 = 1 is not target smoothing's stream
    for other in (_ex().normal(ids, step + 1, A, 9), _ex().normal(ids, step, A, 10),
                  _ex().normal([i + 1 for i in ids], step, A, 9)):
        assert not np.any(other == z)
    ts = np.stack([tn.normal(A, 9, i, step) for i in ids])
    assert not np.any(np.isclose(ts, want, rtol=0, atol=1e-12))


def test_zero_crossings_of_sincospi_are_exact():
    s, c = _ex()._sincospi(np.array([0.5, 1.0, 1.5, 0.25, 2.0 - 2 ** -23]))
    assert c[0] == 0 and s[1] == 0 and c[2] == 0 and s[0] == 1 and c[1] == -1 and s[2] == -1
    assert np.allclose(s, np.sin(np.pi * np.array([0.5, 1.0, 1.5, 0.25, 2.0 - 2 ** -23])), atol=1e-15)


@pytest.mark.parametrize("mode", ["gaussian", "ou"])
def test_host_noise_against_float64_with_episode_resets(mode):
    """200 steps of 5 lanes with staggered episode starts: fp32 HostNoise against the float64 recurrence."""
    ex = _ex()
    ids, A, T = [3, 0, 11, 7, 15], 6, 200
    o = ex.Exploration(mode, 0.4, 0.05, 16, theta=0.15, seed=2)
    noise = ex.HostNoise(o, ids, A)
    rng = np.random.default_rng(1)
    mu = rng.uniform(-0.9, 0.9, (T, len(ids), A)).astype(np.float32)
    resets = {t: [n for n in range(len(ids)) if t % 37 == (11 * n) % 37] for t in range(1, T)}
    got = np.empty_like(mu)
    for t in range(T):
        noise.reset(resets.get(t, []))
        got[t] = noise.actions(mu[t], t)
    want = xo.run(mu, o.sigmas(ids), ids, 2, mode, theta=0.15, resets=resets)
    assert got.dtype == np.float32
    np.testing.assert_allclose(got, want, rtol=0, atol=2e-6)
    if mode == "ou":                                   # x at a reset is zero: that step's noise is sigma z alone
        lane = 1
        t = next(t for t, lanes in resets.items() if lane in lanes)
        assert np.array_equal(noise.x.shape, (len(ids), A))
        noise2 = ex.HostNoise(o, ids, A)
        first = noise2.actions(np.zeros_like(mu[0]), t)[lane]
        assert np.array_equal(first, np.clip(o.sigmas(ids)[lane] * ex.normal(ids, t, A, 2)[lane], -1, 1))


def test_host_noise_refuses_reference():
    ex = _ex()
    with pytest.raises(ValueError, match="reference"):
        ex.HostNoise(ex.Exploration(), [0], 2)


# ------------------------------------------------------------------------------------------------ 4. Actor vs pool
@pytest.fixture
def dirs(monkeypatch, tmp_path):
    monkeypatch.setenv("R2D2_OBS_SIZE", "5")
    monkeypatch.setenv("R2D2_N_ACTIONS", "3")
    monkeypatch.setenv("R2D2_HIDDEN", "32")
    from actor_pool import initial_model_dict
    torch.manual_seed(0)
    md = initial_model_dict(5, 3, 32)
    for sd in md.values():
        sd["l3.weight"].uniform_(-0.5, 0.5)
    out = []
    for name in ("actor", "pool"):
        d = tmp_path / name
        os.makedirs(d / "memory_data")
        os.makedirs(d / "model_data")
        torch.save(md, d / "model_data" / "model.pt")
        out.append(d)
    return out


def _episodes(path):
    from replay_memory import pack_episode
    payload = torch.load(path, weights_only=False)
    return [pack_episode(rows, states, hidden=32)[:4] for rows, states in
            zip(payload["replay_memory"], payload["recurrent_state"])]


@pytest.mark.parametrize("mode", ["gaussian", "ou"])
def test_actor_and_one_lane_pool_write_the_same_episodes(dirs, monkeypatch, mode):
    """Both step batch-1 models.py nets on the same weights and draw HostNoise at the same t, so obs, actions and
    terminals are identical bit for bit; equal obs and actions make the env's raw rewards equal, and the stored n-step
    sums agree to float32 rounding (the two compute them in different code)."""
    from actor import Actor
    from actor_pool import ActorPool, ModelsStepper
    monkeypatch.setenv("R2D2_EXPLORATION", mode)
    monkeypatch.setenv("R2D2_EXPLORATION_SIGMA", "0.5")
    monkeypatch.setenv("R2D2_EXPLORATION_SIGMA_MIN", "0.1")
    monkeypatch.setenv("R2D2_EXPLORATION_ACTORS", "8")
    monkeypatch.setenv("R2D2_EXPLORATION_SEED", "3")
    aid, E = 5, 64
    monkeypatch.chdir(dirs[0])
    actor = Actor(aid)
    actor.env.episode_len = E
    actor.run(max_episodes=4)
    monkeypatch.chdir(dirs[1])
    pool = ActorPool([aid], stepper=ModelsStepper(5, 3, 32, 1, max_episode_steps=80), seed=1,
                     priority_fn=lambda md, eps: ([np.ones(len(e[0]) - 65, np.float32) for e in eps],
                                                  [_nstep(e[2]) for e in eps]))
    pool.envs[0].episode_len = E
    pool.run(max_steps=4 * E)
    a = _episodes(dirs[0] / "memory_data" / f"memory{aid}.pt")
    p = _episodes(dirs[1] / "memory_data" / f"memory{aid}.pt")
    assert len(a) == len(p) == 4
    for (oa, aa, ra, ta), (op, ap, rp, tp) in zip(a, p):
        assert np.array_equal(oa, op) and np.array_equal(aa, ap) and np.array_equal(ta, tp)
        np.testing.assert_allclose(ra, rp, rtol=1e-6, atol=1e-7)
    acts = np.concatenate([e[1][:E] for e in a])
    assert np.all(np.abs(acts) <= 1) and len(np.unique(acts)) > 100


def _nstep(raw, n=5, gamma=0.997):
    raw = np.asarray(raw, np.float64)
    out = raw.copy()
    for i in range(len(raw) - n):
        out[i] = sum(raw[i + j] * gamma ** j for j in range(n))
    return out.astype(np.float32)


def test_reference_mode_keeps_its_noise_sources(dirs, monkeypatch):
    """ActorPool: clip(mu + rng.normal(0, noise_std)) from its seeded generator; Actor: numpy's global state."""
    from actor import Actor
    from actor_pool import ActorPool, ModelsStepper
    for k in [k for k in os.environ if k.startswith("R2D2_EXPLORATION")]:
        monkeypatch.delenv(k)
    monkeypatch.chdir(dirs[1])
    pool = ActorPool([2, 4], stepper=ModelsStepper(5, 3, 32, 2), seed=7, noise_std=0.3,
                     priority_fn=lambda md, eps: ([], []))
    rng = np.random.default_rng(7)
    for _ in range(3):
        pool.step()
        want = np.clip(pool.last_mu + rng.normal(0.0, 0.3, pool.last_mu.shape), -1, 1).astype(np.float32)
        got = np.stack([pool.sequence[lane][-1][1] for lane in range(2)])
        assert np.array_equal(got, want)
    assert pool.stepper.actions is None
    monkeypatch.chdir(dirs[0])
    actor = Actor(2)
    actor.env.episode_len = 3
    np.random.seed(11)
    actor.run(max_episodes=1)
    assert actor.noise is None
    first_obs = actor.sequence[0][0]
    with torch.no_grad():
        for _, net in actor._nets():
            net.reset_state()
        mu = actor.actor(torch.from_numpy(first_obs[None])).numpy()[0]
    want = np.clip(mu + np.random.RandomState(11).normal(0, 0.3, 3), -1, 1).astype(np.float32)
    assert np.array_equal(actor.sequence[0][1], want)


# ------------------------------------------------------------------------------------------------ 5. compiler report
KERNEL = "policy_explore_head_kernel"


def test_explore_head_kernel_does_not_spill():
    report, stderr = ptxas_report("policy.cu")
    found = 0
    for m in report:
        if KERNEL in m.group(1):
            found += 1
            assert m.group(2) == m.group(3) == m.group(4) == "0", m.group(0)
    assert found == 2, stderr[-2000:]


def test_explore_head_sass_has_no_local_memory():
    funcs = functions(library_sass(), KERNEL)
    assert len(funcs) == 2, sorted(funcs)
    for name, body in funcs.items():
        body_ops = [op for op, _ in ops(body)]
        assert not [op for op in body_ops if op.startswith(("LDL", "STL"))], f"local-memory traffic in {name}"
        assert any(op.startswith("FFMA") for op in body_ops), name
        assert "IMAD.HI.U32" in body_ops or any(op.startswith("IMAD.WIDE.U32") for op in body_ops), name

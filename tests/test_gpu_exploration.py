"""r2d2_policy_step_explore on the H100: mu, mu_t and the states bitwise those of the plain step; the noise of a zeroed
actor head against the float64 generator; c3 = 1 apart from target smoothing's streams; lane independence through
ActorPool; OU over 100 steps with episode resets; PolicyStepper against ModelsStepper; and every refused argument
launching nothing."""
import os
from ctypes import c_void_p

import numpy as np
import pytest
import torch

import exploration_oracle as xo
from oracle.actor_oracle import policy_params

pytestmark = pytest.mark.gpu

O = 24


def _stepper(A, H, N, seed, max_episode_steps=4):
    from r2d2_b200.policy_step import PolicyStepper
    st = PolicyStepper(O, A, H, N, device="cuda", max_episode_steps=max_episode_steps)
    st.load(policy_params(O, A, H, seed))
    return st


def _zero_actor_head(st, A, H):
    """W3 and b3 of the actor are the block's last A H + A floats: mu = tanh(0) = 0 exactly."""
    st.params[0][-(A * H + A):].zero_()


def _ulp_bound(want, k):
    """k ulp of float32 at |want| (float64 values)."""
    return k * np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)


def _explore(kind, seed, step, ids, sigma, ou_state=None, omt=0.85):
    return dict(mode=kind, seed=seed, step=step, one_minus_theta=omt,
                actor_id=torch.tensor(ids, dtype=torch.int32, device="cuda"),
                sigma=torch.tensor(sigma, dtype=torch.float32, device="cuda"), ou_state=ou_state)


SHAPES = [(H, A, N) for H in (32, 128, 512) for A in (1, 6, 17, 64) for N in (1, 16, 17, 256)]


@pytest.mark.parametrize("norm", [False, True], ids=["raw", "obs_norm"])
@pytest.mark.parametrize("H,A,N", SHAPES)
def test_explore_step(H, A, N, norm):
    from r2d2_b200.exploration import normal
    from r2d2_b200.policy_step import policy_step
    st = _stepper(A, H, N, seed=H + A + N)
    g = torch.Generator(device="cuda").manual_seed(N)
    obs = torch.randn((N, O), device="cuda", generator=g)
    s_in = 0.5 * torch.randn((4, 2, N, H), device="cuda", generator=g)
    obs_norm = (torch.randn(O, device="cuda", generator=g), torch.rand(O, device="cuda", generator=g) + 0.5, 3.0) \
        if norm else None
    ids = [int(i) for i in np.random.default_rng(N).permutation(1000)[:N]]
    sigma = np.random.default_rng(A).uniform(0.02, 0.15, N).astype(np.float32)
    step = 12345 + (2 ** 32 if H == 128 else 0)

    def run(exploration=None, params=None):
        ws = torch.full_like(st.workspace, float("nan"))
        mu = torch.full((N, A), float("nan"), device="cuda")
        out = torch.full_like(s_in, float("nan"))
        act = torch.full((N, A), float("nan"), device="cuda") if exploration else None
        policy_step(params or st.params, obs, s_in, out, mu, ws, obs_norm, exploration=exploration, action=act)
        mu_t = ws[N * H * 20:N * H * 20 + N * A].view(N, A)
        return mu, mu_t, out, act

    # 1. mu, mu_t and every state are the plain step's bits, in both modes
    mu, mu_t, out, _ = run()
    ou = torch.zeros((N, A), device="cuda")
    for ex in (_explore("gaussian", 3, step, ids, sigma), _explore("ou", 3, step, ids, sigma, ou_state=ou)):
        m2, mt2, o2, act = run(ex)
        assert torch.equal(m2, mu) and torch.equal(mt2, mu_t) and torch.equal(o2, out), ex["mode"]
        assert torch.isfinite(act).all() and (act.abs() <= 1).all()
    # 2. a zeroed actor head: mu = 0, action = sigma z (|sigma z| < 1: no clipping) against float64 and the host
    _zero_actor_head(st, A, H)
    mu0, _, out0, act = run(_explore("gaussian", 3, step, ids, sigma))
    assert torch.equal(mu0, torch.zeros_like(mu0))
    got = act.cpu().numpy().astype(np.float64)
    want = sigma[:, None].astype(np.float64) * xo.normal(ids, step, A, 3)
    # Philox words are integers (checked bit for bit against the oracle on the host); z is within 3 ulp after the
    # device's logf and sincospif (1 ulp each), sigma z adds one rounding: 4 ulp of the float64 product
    assert np.all(np.abs(got - want) <= _ulp_bound(want, 4)), np.max(np.abs(got - want) / _ulp_bound(want, 1))
    # the host restatement is within 2.5 ulp of the float64 product and the device within 4: 8 ulp between them
    host = sigma[:, None] * normal(ids, step, A, 3)
    assert np.all(np.abs(got - host) <= _ulp_bound(want, 8)), np.max(np.abs(got - host) / _ulp_bound(want, 1))
    # the OU state after one step from zero is the same sigma z, written back
    ou.zero_()
    _, _, _, act_ou = run(_explore("ou", 3, step, ids, sigma, ou_state=ou))
    assert torch.equal(act_ou, act) and torch.equal(ou, act)


def test_streams_differ_from_target_smoothing():
    """Equal (seed, actor id = rank, step = iter): the exploration stream (c3 = 1) shares no value with target
    smoothing's (c3 = 0)."""
    from r2d2_b200 import native as nv
    from r2d2_b200.policy_step import policy_step
    A, H, N = 64, 32, 16
    st = _stepper(A, H, N, seed=1)
    _zero_actor_head(st, A, H)
    ids = list(range(100, 100 + N))
    act = torch.empty((N, A), device="cuda")
    policy_step(st.params, torch.zeros((N, O), device="cuda"), torch.zeros((4, 2, N, H), device="cuda"),
                torch.empty((4, 2, N, H), device="cuda"), torch.empty((N, A), device="cuda"), st.workspace,
                exploration=_explore("gaussian", 9, 77, ids, [0.1] * N), action=act)
    zero = torch.zeros(A, device="cuda")
    for n, i in enumerate(ids):
        ts = torch.empty(A, device="cuda")
        nv.check(nv.lib().r2d2_target_smoothing(nv.dptr(zero), nv.dptr(ts), A, 0.1, 3e38, 9, i, 77,
                                                nv.current_stream()))
        assert not torch.any(ts == act[n]), n


@pytest.fixture
def pool_dir(monkeypatch, tmp_path):
    monkeypatch.setenv("R2D2_OBS_SIZE", str(O))
    monkeypatch.setenv("R2D2_N_ACTIONS", "6")
    monkeypatch.setenv("R2D2_HIDDEN", "128")
    monkeypatch.chdir(tmp_path)
    os.makedirs("memory_data")
    os.makedirs("model_data")
    from actor_pool import initial_model_dict
    torch.manual_seed(0)
    md = initial_model_dict(O, 6, 128)
    torch.save(md, "model_data/model.pt")
    return md


@pytest.mark.parametrize("mode", ["gaussian", "ou"])
def test_pool_lanes_are_independent(pool_dir, monkeypatch, mode):
    from actor_pool import ActorPool
    monkeypatch.setenv("R2D2_EXPLORATION", mode)
    monkeypatch.setenv("R2D2_EXPLORATION_SIGMA", "0.4")
    monkeypatch.setenv("R2D2_EXPLORATION_SIGMA_MIN", "0.05")
    monkeypatch.setenv("R2D2_EXPLORATION_ACTORS", "32")
    ids = [3, 17, 0, 31, 8]

    def actions(pool_ids, steps=40):
        from utils import get_obs
        pool = ActorPool(pool_ids, device="cuda", priority_fn=lambda md, eps: ([], []))
        # the pool resets lane 0's env once more at construction (to read the obs size, as Actor.__init__ does): give
        # every env that history, so an id's env starts from the same obs in every lane
        for lane in range(1, len(pool_ids)):
            pool.obs[lane] = get_obs(pool.envs[lane].reset().observation)[0]
        for env in pool.envs:
            env.episode_len = 13 + env.n_actions          # episodes end and restart inside the window
        out = []
        for _ in range(steps):
            pool.step()
            out.append(pool.stepper.actions.copy())
            assert np.array_equal(np.stack([pool.sequence[k][-1][1] if pool.sequence[k] else out[-1][k]
                                            for k in range(len(pool_ids))]), out[-1])
        return {i: np.stack([a[k] for a in out]) for k, i in enumerate(pool_ids)}

    base = actions(ids)
    perm = actions(ids[::-1])
    for i in ids:
        assert np.array_equal(base[i], perm[i]), i
    for i in (17, 31):
        assert np.array_equal(base[i], actions([i])[i]), i


def test_ou_over_episodes_against_float64():
    """100 steps, zeroed head (mu = 0): actions are clip(x) with x the float64 OU recurrence, lanes reset on their own
    schedule; reset zeroes a lane's x exactly."""
    from r2d2_b200.exploration import Exploration
    A, H, N, T = 6, 64, 17, 100
    st = _stepper(A, H, N, seed=2, max_episode_steps=T)
    _zero_actor_head(st, A, H)
    ids = list(range(40, 40 + N))
    opt = Exploration("ou", 0.5, 0.05, 64, theta=0.15, seed=5)
    st.set_exploration(opt, ids)
    st.reset(range(N))
    resets = {t: [n for n in range(N) if t % 23 == (5 * n) % 23] for t in range(1, T)}
    got = np.empty((T, N, A), np.float32)
    obs = np.random.default_rng(0).standard_normal((N, O)).astype(np.float32)
    for t in range(T):
        if resets.get(t):
            st.reset(resets[t])
            assert not st.exploration["ou_state"][resets[t]].any()
            assert st.exploration["ou_state"].abs().sum() > 0
        st.step(obs)
        got[t] = st.actions
    want = xo.run(np.zeros((T, N, A)), opt.sigmas(ids), ids, 5, "ou", theta=0.15, resets=resets)
    # fp32 recurrence with fl32(1 - theta) against float64: the error stays below 1e-5 in absolute terms
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-5)


@pytest.mark.parametrize("mode", ["gaussian", "ou"])
def test_policy_stepper_matches_models_stepper(mode):
    from actor_pool import ModelsStepper
    from r2d2_b200.exploration import Exploration
    A, H, N = 6, 128, 16
    md = {k: {n: torch.from_numpy(v) for n, v in sd.items()} for k, sd in policy_params(O, A, H, seed=8).items()}
    ids = list(range(N))[::-1]
    opt = Exploration(mode, 0.3, 0.05, N, seed=1)
    gpu = _stepper(A, H, N, seed=8, max_episode_steps=64)
    cpu = ModelsStepper(O, A, H, N, max_episode_steps=64)
    cpu.load(md)
    rng = np.random.default_rng(3)
    for st in (gpu, cpu):
        st.set_exploration(opt, ids)
        st.reset(range(N))
    for t in range(60):
        if t == 30:
            for st in (gpu, cpu):
                st.reset([2, 9])
        obs = rng.standard_normal((N, O)).astype(np.float32)
        mg, mc = gpu.step(obs), cpu.step(obs)
        np.testing.assert_allclose(mg, mc, atol=1e-4)
        np.testing.assert_allclose(gpu.actions, cpu.actions, atol=1e-4)


def test_refused_arguments_launch_nothing():
    from r2d2_b200 import native as nv
    lib = nv.lib()
    A, H, N = 6, 64, 8
    st = _stepper(A, H, N, seed=4)
    dev = lambda *s: torch.zeros(s, device="cuda")  # noqa: E731
    obs, s_in, s_out, mu, act, ou = dev(N, O), dev(4, 2, N, H), dev(4, 2, N, H), dev(N, A), dev(N, A), dev(N, A)
    big = dev(2 * N * A)
    ids = torch.arange(N, dtype=torch.int32, device="cuda")
    good_sigma = torch.full((N,), 0.1, device="cuda")
    ptrs = (c_void_p * 4)(*[nv.dptr(p).value for p in st.params])

    def call(shape=(O, A, H), n=N, action=act, mu_=mu, **kw):
        f = dict(kind=nv.EXPLORATION_OU, seed=0, step=0, one_minus_theta=0.85, actor_id=nv.dptr(ids, torch.int32),
                 sigma=nv.dptr(good_sigma), ou_state=nv.dptr(ou))
        f.update(kw)
        ex = nv.Exploration(**f)
        return lib.r2d2_policy_step_explore(nv.byref(nv.NetShape(*shape, 0)), ptrs, nv.dptr(obs), nv.dptr(s_in),
                                            nv.dptr(s_out), nv.dptr(mu_), n, nv.dptr(st.workspace), None, None, 0.0,
                                            nv.byref(ex), action, nv.current_stream())

    assert call(action=nv.dptr(act)) == 0
    torch.cuda.synchronize()
    bad_sigmas = [torch.tensor([0.1] * (N - 1) + [v], device="cuda") for v in (float("nan"), -0.5, float("inf"))]
    cases = [dict(kind=2), dict(kind=-1), dict(actor_id=None), dict(sigma=None), dict(ou_state=None),
             dict(kind=nv.EXPLORATION_GAUSSIAN), dict(one_minus_theta=1.0), dict(one_minus_theta=-0.1),
             dict(one_minus_theta=float("nan")), dict(action=None), dict(action=nv.dptr(mu)),
             dict(action=nv.dptr(big[1:1 + N * A]), mu_=big[:N * A])] + [dict(sigma=nv.dptr(s)) for s in bad_sigmas]
    for kw in cases:
        kw.setdefault("action", nv.dptr(act))
        before = lib.r2d2_launch_count()
        rc = call(**kw)
        assert rc == -2 and lib.r2d2_launch_count() == before, (kw, rc, lib.r2d2_last_error())
    for shape, n in (((O, 65, H), N), ((O, A, 48), N), ((O, A, H), 257), ((O, A, H), 0)):
        before = lib.r2d2_launch_count()
        assert call(shape=shape, n=n, action=nv.dptr(act)) == -3 and lib.r2d2_launch_count() == before
    before = lib.r2d2_launch_count()
    assert lib.r2d2_policy_step_explore(nv.byref(nv.NetShape(O, A, H, 0)), ptrs, nv.dptr(obs), nv.dptr(s_in),
                                        nv.dptr(s_out), nv.dptr(mu), N, nv.dptr(st.workspace), None, None, 0.0, None,
                                        nv.dptr(act), nv.current_stream()) == -2
    assert lib.r2d2_launch_count() == before
    with pytest.raises(nv.NativeError, match="sigma"):
        nv.check(call(sigma=nv.dptr(bad_sigmas[0]), action=nv.dptr(act)))

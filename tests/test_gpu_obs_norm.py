"""Observation normalisation on the H100: the ingest moments against float64, the merge against the host oracle, the
normalising gathers and policy step against the float32 transform bit for bit, the learner fed normalised batches by the
replay against the learner fed batches normalised by r2d2_obs_normalize, resume, and the drop-in learner and actors."""
import os

import numpy as np
import pytest

from learner_harness import (REPLAY, SMALL, assert_same_bits, episode, gather_out, golden_case, snapshot,
                             trained_dropin_learner)
from obs_norm_oracle import episode_rows, merge, moments, normalize, pair

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

from r2d2_b200 import engine as E  # noqa: E402
from r2d2_b200 import native as nv  # noqa: E402
from r2d2_b200.obs_norm import ObsNormStats  # noqa: E402


def _cfg(O, **kw):
    return E.PathConfig(**dict(dict(obs=O, act=2, hidden=32, batch=8, burn_in=2, learning=4, n_step=2), **kw))


def _episodes(rng, cfg, n, lo=20, hi=60):
    eps = []
    for _ in range(n):
        e = list(episode(rng, cfg, int(rng.integers(lo, hi))))
        e[0] = (e[0] * rng.uniform(0.1, 30, cfg.obs) + rng.uniform(-100, 100, cfg.obs)).astype(np.float32)
        eps.append(tuple(e))
    return eps


def _ingest(cfg, eps, cap, **rk):
    stats = ObsNormStats(cfg.obs, 5.0, "cuda")
    rp = E.DeviceReplay(E.PathConfig(**dict(cfg.__dict__, **rk)), capacity_rows=cap)
    rp.add_episodes(eps, obs_norm=stats)
    torch.cuda.synchronize()
    return rp, stats


def _close(got, ref):
    assert got[0] == ref[0]
    O = (ref.size - 1) // 2
    np.testing.assert_allclose(got[1:1 + O], ref[1:1 + O], rtol=1e-12, atol=1e-12 * max(1.0, np.abs(ref[1:1 + O]).max()))
    np.testing.assert_allclose(got[1 + O:], ref[1 + O:], rtol=1e-12, atol=1e-300)


@pytest.mark.parametrize("O", [1, 3, 17, 376])
def test_ingest_moments_match_float64(O):
    """Several episodes per call, pad rows left out; the call is wider than the ring and wraps onto its own episodes."""
    cfg = _cfg(O)
    rng = np.random.default_rng(O)
    eps = _episodes(rng, cfg, 9)
    total = sum(len(e[0]) for e in eps)
    rp, stats = _ingest(cfg, eps, cap=150)
    assert total > 150 and rp.stats()["n_episodes"] < 9              # the call overwrote its own rows
    _close(stats.ingest_block.cpu().numpy(), moments(episode_rows(eps, cfg.n_step)))
    assert np.array_equal(stats.pending.cpu().numpy(), stats.ingest_block.cpu().numpy())
    _, again = _ingest(cfg, eps, cap=150)                             # two runs, the same bits
    assert torch.equal(again.ingest_block, stats.ingest_block)
    rp.close()


def test_nonfinite_rows_are_left_out_and_counted():
    cfg = _cfg(17)
    rng = np.random.default_rng(3)
    eps = _episodes(rng, cfg, 4)
    eps[0][0][3, 5] = np.nan
    eps[1][0][0, 0] = np.inf
    eps[2][0][7, 16] = -np.inf
    eps[3][0][-1, 2] = np.nan                                          # a pad row: not counted, not used
    rp, stats = _ingest(cfg, eps, cap=4000)
    assert stats.nonfinite_rows == 3
    _close(stats.ingest_block.cpu().numpy(), moments(episode_rows(eps, cfg.n_step)))
    rp.close()


def test_one_call_wider_than_the_row_kernel_grid():
    """70 episodes of 255 rows (17,850 rows) in one call: more rows than one warp per row of the capped grid covers, a
    non-finite row near the end counted."""
    cfg = _cfg(17, burn_in=40, learning=80, n_step=5)
    rng = np.random.default_rng(70)
    eps = []
    for _ in range(70):
        e = list(episode(rng, cfg, 250))
        e[0] = (e[0] * 4 - 7).astype(np.float32)
        eps.append(tuple(e))
    eps[69][0][200, 3] = np.nan
    assert sum(len(e[0]) for e in eps) > 17000
    rp, stats = _ingest(cfg, eps, cap=20000)
    assert stats.nonfinite_rows == 1
    _close(stats.ingest_block.cpu().numpy(), moments(episode_rows(eps, cfg.n_step)))
    rp.close()


@pytest.mark.parametrize("W", [1, 2, 4])
def test_merge_matches_oracle(W):
    rng = np.random.default_rng(W)
    O = 37
    blocks = [moments(rng.standard_normal((int(rng.integers(1, 90)), O)) * 4 + 2) for _ in range(W)]
    if W > 1:
        blocks[1] = np.zeros(1 + 2 * O)                                # a rank that ingested nothing
    start = moments(rng.standard_normal((50, O)))
    running = torch.tensor(start, dtype=torch.float64, device="cuda")
    dev = torch.tensor(np.stack(blocks), dtype=torch.float64, device="cuda")
    mf, sf = torch.empty(O, device="cuda"), torch.empty(O, device="cuda")
    nv.check(nv.lib().r2d2_obs_norm_merge(nv.dptr(running, torch.float64), nv.dptr(dev, torch.float64), W, O,
                                          nv.dptr(mf), nv.dptr(sf), nv.current_stream()))
    ref = start
    for b in blocks:
        ref = merge(ref, b)
    assert np.array_equal(running.cpu().numpy(), ref)
    m, s = pair(ref)
    assert np.array_equal(mf.cpu().numpy(), m) and np.array_equal(sf.cpu().numpy(), s)


def test_ranks_with_different_shards_end_with_identical_statistics():
    cfg = _cfg(17)
    rng = np.random.default_rng(8)
    a = _ingest(cfg, _episodes(rng, cfg, 3), 4000)
    b = _ingest(cfg, _episodes(rng, cfg, 6), 4000)
    blocks = torch.stack([a[1].pending, b[1].pending])
    for _, st in (a, b):
        st.exchange(blocks.clone())
    assert torch.equal(a[1].running, b[1].running) and torch.equal(a[1].mean_f, b[1].mean_f)
    assert torch.equal(a[1].inv_std_f, b[1].inv_std_f) and not a[1].pending.any()


@pytest.mark.parametrize("tier,dtype", [("device", "float32"), ("device", "float16"), ("host", "float32"),
                                        ("host", "float16")])
@pytest.mark.parametrize("O", [17, 376])
def test_gathered_obs_are_the_transform_of_the_raw_rows(tier, dtype, O):
    from learner_harness import draw
    cfg = _cfg(O)
    rng = np.random.default_rng(11)
    rp, stats = _ingest(cfg, _episodes(rng, cfg, 12), 4000, replay_state_dtype=dtype, replay_state_memory=tier)
    stats.clip = 1.5                                                   # some values clamp
    stats.exchange()
    u = torch.rand(64, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    m, s = stats.mean_f.cpu().numpy(), stats.inv_std_f.cpu().numpy()
    for kind in ("plain", "weighted", "chosen"):
        leaf = None
        if kind == "chosen":
            leaf = draw(rp, cfg, "plain", u=u)["leaf"]
            leaf = torch.tensor(leaf, device="cuda")
        rp.attach_obs_norm(stats)
        got = draw(rp, cfg, kind, u=u, leaf=leaf)
        rp.attach_obs_norm(None)
        raw = draw(rp, cfg, kind, u=u, leaf=leaf)
        assert np.array_equal(got["obs"].view(np.uint32), normalize(raw["obs"], m, s, 1.5).view(np.uint32)), kind
        for k in raw:
            if k != "obs":
                assert np.array_equal(got[k], raw[k]), (kind, k)
    rp.close()


@pytest.mark.parametrize("N", [1, 64, 256])
def test_policy_step_ex_equals_policy_step_on_normalised_obs(N):
    from r2d2_b200.policy_step import policy_step
    O, A, H = 376, 17, 128
    g = torch.Generator(device="cuda").manual_seed(N)
    lib = nv.lib()
    params = [torch.randn(lib.r2d2_net_param_count(nv.byref(nv.NetShape(O, A, H, int(k >= 2)))), device="cuda",
                          generator=g) * 0.05 for k in range(4)]
    obs = torch.randn(N, O, device="cuda", generator=g) * 20 + 3
    obs[0, :4] = torch.tensor([float("nan"), float("inf"), -float("inf"), 0.0])
    mean = torch.randn(O, device="cuda", generator=g)
    inv = torch.rand(O, device="cuda", generator=g) * 0.5 + 0.01
    state = torch.randn(4, 2, N, H, device="cuda", generator=g) * 0.1
    pre = torch.empty_like(obs)
    nv.check(lib.r2d2_obs_normalize(nv.dptr(obs), nv.dptr(pre), N, O, nv.dptr(mean), nv.dptr(inv), 5.0,
                                    nv.current_stream()))
    outs = []
    for x, norm in ((pre, None), (obs, (mean, inv, 5.0))):
        so, mu = torch.empty_like(state), torch.empty(N, A, device="cuda")
        policy_step(params, x, state, so, mu, obs_norm=norm)
        outs.append((so, mu))
    torch.cuda.synchronize()
    ref = normalize(obs.cpu().numpy(), mean.cpu().numpy(), inv.cpu().numpy(), 5.0)
    got = pre.cpu().numpy()
    nan = np.isnan(ref)                      # the device's arithmetic returns its canonical NaN, not the input's payload
    assert np.array_equal(np.isnan(got), nan) and nan.any()
    assert np.array_equal(got[~nan].view(np.uint32), ref[~nan].view(np.uint32))
    for a, b in zip(outs[0], outs[1]):                # lane 0 is NaN throughout: compare the bits
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


CFG2 = dict(obs=17, act=6, hidden=256, batch=256, burn_in=40, learning=80, n_step=5)
SHAPES = {"replay": lambda: REPLAY, "cfg2": lambda: CFG2, "walker": lambda: golden_case("ref_walker_h128.npz")[0]}


def _fed_run(norm_in_replay, shape="replay", steps=5, **extra):
    """Pipelined replay-fed run: obs_norm on (the gather normalises), or off with each drawn batch normalised in place
    by r2d2_obs_normalize with statistics computed the same way."""
    cfg = E.PathConfig(**dict(SHAPES[shape](), obs_norm=norm_in_replay, **extra))
    rng = np.random.default_rng(5)
    eps = _episodes(rng, cfg, 24, cfg.rows + 40, cfg.rows + 80)
    rp = E.DeviceReplay(cfg, capacity_rows=24 * (cfg.rows + 80))
    eng = E.LearnerEngine(cfg, seed=7)
    stats = eng.obs_norm if norm_in_replay else ObsNormStats(cfg.obs, cfg.obs_norm_clip, "cuda")
    if norm_in_replay:
        rp.attach_obs_norm(stats)
    rp.add_episodes(eps[:10], obs_norm=stats)
    rp.add_episodes(eps[10:], obs_norm=stats)
    stats.exchange()
    gen = torch.Generator(device="cuda").manual_seed(11)

    def fill(e):
        rp.sample_into(e, generator=gen)
        if not norm_in_replay:
            nv.check(nv.lib().r2d2_obs_normalize(nv.dptr(e.obs), nv.dptr(e.obs), cfg.rows * cfg.batch, cfg.obs,
                                                 nv.dptr(stats.mean_f), nv.dptr(stats.inv_std_f), stats.clip,
                                                 nv.current_stream()))

    def hook(e, used):
        rp.update_priorities(used.leaf_idx, used.priority)
        fill(e)

    fill(eng)
    for _ in range(steps):
        eng.step(prefetch=hook)
    out = snapshot(eng)
    out["running"] = stats.running.clone()
    out["launches"] = torch.tensor(eng.launches_per_iteration)
    rp.close()
    eng.close()
    return out


@pytest.mark.parametrize("shape,extra", [("replay", {}), ("cfg2", {}), ("walker", {}),
                                         ("replay", dict(twin_critic=True, value_rescaling="invertible",
                                                         priority_metric="abs", is_exponent=0.6, priority_exponent=0.9))])
def test_learner_on_normalised_gathers_equals_learner_on_normalised_batches(shape, extra):
    steps = 3 if shape == "cfg2" else 5
    a, b = _fed_run(True, shape, steps, **extra), _fed_run(False, shape, steps, **extra)
    assert a["running"][0] > 0
    assert_same_bits(a, b)


def test_snapshot_resume_continues_bit_for_bit(tmp_path):
    """Replay-fed sequential steps, an ingest and its exchange, then the training state and a replay snapshot (with the
    CUDA RNG); a fresh engine and shard restored from both continue with the same bits as the run that went on - every
    batch after the resume gathered through the restored statistics."""
    cfg = E.PathConfig(**REPLAY, obs_norm=True)
    rng = np.random.default_rng(12)
    eps = _episodes(rng, cfg, 24, cfg.rows + 40, cfg.rows + 80)

    def make(seed):
        eng = E.LearnerEngine(cfg, seed=seed)
        rp = E.DeviceReplay(cfg, capacity_rows=24 * (cfg.rows + 80))
        rp.attach_obs_norm(eng.obs_norm)
        return eng, rp

    def step(eng, rp):                                   # run_loop's sequential step
        rp.sample_into(eng)
        eng.step()
        rp.update_priorities(eng.leaf_idx, eng.priority)

    a, rpa = make(7)
    rpa.add_episodes(eps[:12], obs_norm=a.obs_norm)
    a.obs_norm.exchange()
    torch.manual_seed(3)
    for _ in range(2):
        step(a, rpa)
    rpa.add_episodes(eps[12:], obs_norm=a.obs_norm)
    a.obs_norm.exchange()
    st = a.training_state()
    assert st["obs_norm"]["n"] > 0 and st["obs_norm"]["mean"].dtype == np.float64 and st["obs_norm"]["clip"] == 5.0
    path = str(tmp_path / "shard0of1")
    rpa.save_snapshot(path)
    for _ in range(3):
        step(a, rpa)
    b, rpb = make(123)                                   # other initial weights: everything comes from the state
    b.load_training_state(st)
    rpb.load_snapshot(path)                              # restores the CUDA RNG that draws the next batch
    for k in ("running", "mean_f", "inv_std_f"):
        assert torch.equal(getattr(a.obs_norm, k), getattr(b.obs_norm, k)), k
    for _ in range(3):
        step(b, rpb)
    assert_same_bits(snapshot(a), snapshot(b))
    off = E.LearnerEngine(E.PathConfig(**REPLAY), seed=1)
    with pytest.raises(ValueError, match="obs_norm"):
        off.load_training_state(st)
    other_clip = E.LearnerEngine(E.PathConfig(**REPLAY, obs_norm=True, obs_norm_clip=3.0), seed=1)
    with pytest.raises(ValueError, match="clip"):
        other_clip.load_training_state(st)
    for x in (rpa, rpb, a, b, off, other_clip):
        x.close()


def test_global_draw_normalises_and_replicas_stay_identical():
    """Two in-process ranks with different shards, global sampling: the ranks merge each other's pending blocks in
    rank order and end with the same statistics; the owner-side gathers into both ranks' slots write the transform of
    the owners' raw rows; the replicas stay bit-identical."""
    from global_harness import GlobalRun
    kw = dict(SMALL, hidden=64, target_interval=3, obs_norm=True)
    run = GlobalRun(E, 2, kw, seed=1)
    engs = run.g.engines
    for r, eng in enumerate(engs):                       # each rank's ingests, into its pending block
        scratch = E.DeviceReplay(run.cfg, capacity_rows=20000)
        scratch.add_episodes(run.episodes[r], obs_norm=eng.obs_norm)
        scratch.close()
    blocks = torch.stack([e.obs_norm.pending for e in engs])
    for r, eng in enumerate(engs):
        eng.obs_norm.exchange(blocks.clone())
        run.shards[r].attach_obs_norm(eng.obs_norm)
    for k in ("running", "mean_f", "inv_std_f"):
        assert torch.equal(getattr(engs[0].obs_norm, k), getattr(engs[1].obs_norm, k)), k
    seen = []

    def on_critic(slot):
        seen.append({k: run.slot_cat(k, slot).clone() for k in ("obs", "leaf_idx", "shard")})

    run.run(4, prefetch=True, on_critic=on_critic)
    torch.cuda.synchronize()
    assert run.status() == [0, 0] and seen
    m, s = engs[0].obs_norm.mean_f.cpu().numpy(), engs[0].obs_norm.inv_std_f.cpu().numpy()
    for rp in run.shards:
        rp.attach_obs_norm(None)
    for b in seen:
        obs = b["obs"].cpu().numpy()
        for r, rp in enumerate(run.shards):
            cols = torch.nonzero(b["shard"] == r).flatten()
            if cols.numel() == 0:
                continue
            leaf = b["leaf_idx"][cols].contiguous()
            out = gather_out(run.cfg, leaf.numel())
            nv.check(nv.lib().r2d2_replay_gather(rp._h, nv.dptr(leaf, torch.int64), leaf.numel(), nv.dptr(out["obs"]),
                                                 None, None, None, None, nv.current_stream()))
            torch.cuda.synchronize()
            ref = normalize(out["obs"].cpu().numpy(), m, s, 5.0)
            got = obs[:, cols.cpu().numpy()]
            assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))
    for net in ("actor", "critic", "target_actor", "target_critic"):
        assert torch.equal(engs[0].flat[net], engs[1].flat[net]), net
    for d in ("exp_avg", "exp_avg_sq"):
        for net in ("actor", "critic"):
            assert torch.equal(getattr(engs[0], d)[net], getattr(engs[1], d)[net]), (d, net)
    run.close()


def test_actor_priorities_with_the_key_match_the_oracle_on_normalised_episodes():
    from oracle import actor_oracle
    from r2d2_b200 import actor_priority
    O, A, H = 5, 2, 32
    g = torch.Generator().manual_seed(0)
    from r2d2_b200.engine import init_reference_params
    pc = E.PathConfig(obs=O, act=A, hidden=H)
    critic, tactor, tcritic = (init_reference_params(pc, c, g) for c in (True, False, True))
    rng = np.random.default_rng(4)
    eps = []
    for n in (80, 95):
        obs = (rng.standard_normal((n, O)) * 7 + 3).astype(np.float32)
        eps.append((obs, rng.uniform(-1, 1, (n, A)).astype(np.float32), rng.standard_normal(n).astype(np.float32),
                    np.r_[np.zeros(n - 5), np.ones(5)].astype(np.float32)))
    key = {"mean_f": torch.full((O,), 3.0), "inv_std_f": torch.full((O,), 1 / 7.0), "clip": 2.0}
    got, _ = actor_priority.episode_priorities(critic, tactor, tcritic, eps, hidden=H, obs_norm=key)
    normed = [(normalize(o, key["mean_f"].numpy(), key["inv_std_f"].numpy(), 2.0),) + e[1:]
              for e, o in zip(eps, (e[0] for e in eps))]
    ref, _ = actor_priority.episode_priorities(critic, tactor, tcritic, normed, hidden=H)
    for x, y in zip(got, ref):
        assert np.array_equal(x, y)
    for x, (o, a_, r, d) in zip(got, normed):
        oref = actor_oracle.episode_priorities(critic, tactor, tcritic, o, a_, r, d, burn_in=20, learning=40, n_step=5,
                                               gamma=0.997)
        np.testing.assert_allclose(x, oref, rtol=1e-3, atol=1e-6)


def test_dropin_learner_and_actors_with_obs_norm(monkeypatch):
    with trained_dropin_learner(monkeypatch, R2D2_OBS_NORM="1", R2D2_OBS_NORM_CLIP="4") as (lr, actors):
        st = lr.engine.obs_norm
        assert st.count > 0 and st.clip == 4.0
        lr.save_model()
        md = torch.load(os.path.join("model_data", "model.pt"), map_location="cpu")
        assert set(md) == {"actor", "target_actor", "critic", "target_critic", "obs_norm"}
        assert torch.equal(md["obs_norm"]["mean_f"], st.mean_f.cpu()) and md["obs_norm"]["clip"] == 4.0
        a = actors[0]
        a.load_model()
        assert a.obs_norm is not None
        a.run(max_episodes=1)
        assert lr.engine.training_state()["obs_norm"]["n"] == st.count


def test_policy_stepper_with_the_key_equals_the_stepper_on_normalised_obs():
    from actor_pool import initial_model_dict
    from r2d2_b200.policy_step import PolicyStepper
    O, A, H, N = 376, 17, 128, 64
    torch.manual_seed(1)
    md = initial_model_dict(O, A, H)
    rng = np.random.default_rng(1)
    key = {"mean_f": torch.from_numpy(rng.standard_normal(O).astype(np.float32)),
           "inv_std_f": torch.from_numpy(rng.uniform(0.05, 2, O).astype(np.float32)), "clip": 2.5}
    plain, normed = PolicyStepper(O, A, H, N, device="cuda"), PolicyStepper(O, A, H, N, device="cuda")
    plain.load(md)
    normed.load(dict(md, obs_norm=key))
    assert plain.obs_norm is None and normed.obs_norm is not None
    for t in range(3):
        obs = (rng.standard_normal((N, O)) * 6).astype(np.float32)
        mu_n = normed.step(obs)
        mu_p = plain.step(normalize(obs, key["mean_f"].numpy(), key["inv_std_f"].numpy(), 2.5))
        assert np.array_equal(mu_n.view(np.uint32), mu_p.view(np.uint32)), t
    assert torch.equal(plain.ring.view(torch.int32), normed.ring.view(torch.int32))


def test_actor_pool_runs_with_the_key(tmp_path, monkeypatch):
    """ActorPool following a model.pt with the `obs_norm` entry: its stepper and its priority chains normalise, and it
    writes the usual memory files."""
    from actor_pool import ActorPool, initial_model_dict
    O, A, H = 5, 2, 64
    for k, v in dict(R2D2_OBS_SIZE=str(O), R2D2_N_ACTIONS=str(A), R2D2_HIDDEN=str(H)).items():
        monkeypatch.setenv(k, v)
    monkeypatch.chdir(tmp_path)
    os.makedirs("memory_data")
    os.makedirs("model_data")
    torch.manual_seed(0)
    md = initial_model_dict(O, A, H)
    md["obs_norm"] = {"mean_f": torch.full((O,), 0.1), "inv_std_f": torch.full((O,), 3.0), "clip": 1.0}
    torch.save(md, "model_data/model.pt")
    pool = ActorPool(range(4), device="cuda", noise_std=0.0)
    assert pool.stepper.obs_norm is not None and pool.model_dict["obs_norm"]["clip"] == 1.0
    seen = []
    gpu_prio = pool.priority_fn

    def prio(model_dict, episodes):
        out = gpu_prio(model_dict, episodes)
        seen.append(out)
        return out
    pool.priority_fn = prio
    for env in pool.envs:
        env.episode_len = 70
    pool.run(max_steps=360)
    assert seen and all(np.isfinite(p).all() for out in seen for p in out[0])
    assert any(os.path.isfile("memory_data/memory%d.pt" % i) for i in range(4))

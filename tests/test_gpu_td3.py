"""TD3's target on the GPU: the defaults keep their bits and launches, a twin whose critics are equal behaves like one
critic, the smoothing kernel's noise against the numpy Philox restatement, multi-iteration runs against the float64
TD3 oracle (goldens, cfg-2, rescaling with importance weights, A = 1 and 64), the pipelined / replay-fed / resumed
schedules bit for bit, the data-parallel exchange of the doubled critic block on one GPU, and the drop-in learner."""
import os
import tempfile

import numpy as np
import pytest
import torch

import rescale_oracle as ro
import td3_oracle as t3
from conftest import golden_batch, golden_params, load_golden, rel_l2
from oracle import ref_port
from peer_harness import PeerGroup, split_batch
from test_gpu_prioritized_replay import episode

pytestmark = pytest.mark.gpu

TOL = 1e-3
SMALL = dict(obs=6, act=2, hidden=64, batch=8, burn_in=4, learning=6, n_step=2)
TD3 = dict(twin_critic=True, target_noise=0.2, target_noise_clip=0.5)


@pytest.fixture(scope="module")
def E():
    from r2d2_b200 import engine
    return engine


def _snapshot(eng):
    torch.cuda.synchronize()
    out = {f"flat.{n}": eng.flat[n].clone() for n in ("actor", "critic", "target_actor", "target_critic")}
    for d, name in ((eng.exp_avg, "m"), (eng.exp_avg_sq, "v")):
        out.update({f"{name}.{n}": d[n].clone() for n in ("actor", "critic")})
    out.update({k: getattr(eng, k).clone() for k in ("q_value", "target_q_value", "priority", "losses", "grad_norms")})
    if eng.q_value2 is not None:
        out["q_value2"] = eng.q_value2.clone()
    return out


def _assert_same_bits(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert torch.equal(a[k], b[k]), k


def _np(sd):
    return {k: v.detach().cpu().numpy() for k, v in sd.items()}


# ---------------------------------------------------------------------------------------------------- 1. defaults
def _fixed_run(E, steps=4, setter=None, **extra):
    cfg = E.PathConfig(**SMALL, target_interval=2, **extra)
    eng = E.LearnerEngine(cfg, seed=3)
    if setter:
        setter(eng)
    pc = ref_port.PathConfig(**SMALL)
    for it in range(steps):
        eng.set_batch(ref_port.synthetic_batch(pc, seed=20 + it))
        eng.step()
    out = _snapshot(eng)
    out["launches"] = torch.tensor(eng.launches_per_iteration)
    eng.close()
    return out


def test_defaults_keep_bits_and_launches(E):
    base = _fixed_run(E)
    _assert_same_bits(base, _fixed_run(E, twin_critic=False, target_noise=0.0))
    _assert_same_bits(base, _fixed_run(E, setter=lambda e: e.set_target_smoothing(0.0, 0.5, 0, 0)))
    twin = _fixed_run(E, twin_critic=True)
    smooth = _fixed_run(E, **TD3)
    assert int(smooth["launches"]) == int(twin["launches"]) + 1 > int(base["launches"])   # one smoothing launch
    assert _fixed_run(E, target_noise=0.2)["launches"] == base["launches"] + 1


def test_library_rejects_bad_values(E):
    eng = E.LearnerEngine(E.PathConfig(**SMALL))
    lib = eng.lib
    for sigma, clip in ((-0.1, 0.5), (float("nan"), 0.5), (float("inf"), 0.5), (0.2, 0.0), (0.2, -1.0),
                        (0.2, float("inf")), (0.2, float("nan"))):
        assert lib.r2d2_learner_set_target_smoothing(eng._h, sigma, clip, 0, 0) == -2          # R2D2_ERR_ARG
    assert lib.r2d2_learner_set_target_smoothing(eng._h, 0.2, 0.5, 0, 0) == 0
    pc = ref_port.PathConfig(**SMALL)
    eng.set_batch(ref_port.synthetic_batch(pc, seed=1))
    eng.step(prefetch=lambda e, used: e.set_batch(ref_port.synthetic_batch(pc, seed=2)))   # next targets run ahead
    assert lib.r2d2_learner_set_target_smoothing(eng._h, 0.1, 0.5, 0, 0) == -4              # R2D2_ERR_STATE
    eng.step()
    assert lib.r2d2_learner_set_target_smoothing(eng._h, 0.1, 0.5, 0, 0) == 0
    from r2d2_b200 import native as nv
    bad = nv.LearnerOptions(2)
    h = nv.c_void_p()
    assert lib.r2d2_learner_create_ex(nv.byref(h), nv.byref(nv.LearnerConfig()), nv.byref(bad)) == -2
    eng.close()


def test_twin_memory_is_reported(E):
    a = E.LearnerEngine(E.PathConfig(**SMALL))
    b = E.LearnerEngine(E.PathConfig(**SMALL, twin_critic=True))
    assert a.twin_added_bytes == 0 and b.twin_added_bytes > 0 and a.q_value2 is None
    P = a.flat["critic"].numel()
    assert b._critic2_off % 64 == 0 and P <= b._critic2_off < P + 64 and b.flat["critic"].numel() == 2 * b._critic2_off
    assert len(b.losses) == 3
    a.close()
    b.close()


# ---------------------------------------------------------------------------------------------------- 2. symmetry
def test_equal_twins_behave_like_one_critic(E):
    pc = ref_port.PathConfig(**SMALL)
    batch = ref_port.synthetic_batch(pc, seed=5)
    batch["c_state"][:] = 0
    batch["tc_state"][:] = 0
    twin = E.LearnerEngine(E.PathConfig(**SMALL, twin_critic=True), seed=4)
    one = E.LearnerEngine(E.PathConfig(**SMALL), seed=4)
    twin.load_state_dicts(None, None, critic2=twin.state_dict("critic"), target_critic2=twin.state_dict("target_critic"))
    for e in (twin, one):
        e.set_batch(batch)
        e.step()
    torch.cuda.synchronize()
    P, off = twin._n_critic, twin._critic2_off
    assert torch.equal(twin.q_value2, twin.q_value)
    assert torch.equal(twin.losses[2], twin.losses[0])
    g = twin.grads["critic"]
    assert torch.equal(g[:P], g[off:off + P]) and not g[P:off].any() and not g[off + P:].any()
    assert torch.equal(twin.target_q_value, one.target_q_value)
    assert torch.equal(twin.q_value, one.q_value) and torch.equal(twin.priority, one.priority)
    twin.close()
    one.close()


# ---------------------------------------------------------------------------------------------------- 3. noise
def _device_z(lib, n, seed, rank, it):
    """r2d2_target_smoothing on mu = 0 with sigma = 2^-4: every |sigma z| < 1, so out * 16 is z exactly."""
    from r2d2_b200 import native as nv
    mu = torch.zeros(n, device="cuda")
    out = torch.empty_like(mu)
    nv.check(lib.r2d2_target_smoothing(nv.dptr(mu), nv.dptr(out), n, 0.0625, 1e30, seed, rank, it, nv.current_stream()))
    torch.cuda.synchronize()
    return out.cpu().numpy().astype(np.float64) * 16.0


def test_noise_matches_numpy_philox(E):
    from r2d2_b200 import native as nv
    lib = nv.lib()
    n = (1 << 20) + 3                                    # a partial last group of four
    for seed, rank, it in ((0, 0, 0), (12345, 3, 7), (2 ** 32 - 1, 1, 2 ** 33 + 5)):
        got, want = _device_z(lib, n, seed, rank, it), t3.normal(n, seed, rank, it)
        err = np.abs(got - want) / np.maximum(np.abs(want), 1e-30)
        assert err.max() < 1e-6, (seed, rank, it, float(err.max()))
    base = _device_z(lib, 4096, 5, 0, 1)
    for other in (_device_z(lib, 4096, 5, 1, 1), _device_z(lib, 4096, 5, 0, 2), _device_z(lib, 4096, 6, 0, 1)):
        assert not np.any(other == base)
    from scipy import stats
    res = stats.kstest(_device_z(lib, 1 << 20, 2024, 0, 0), "norm")     # fixed seed: deterministic
    assert res.pvalue > 1e-3, res


def test_noise_clip_and_final_clamp(E):
    from r2d2_b200 import native as nv
    lib = nv.lib()
    n = 1 << 16
    mu = torch.full((n,), 0.9, device="cuda")
    out = torch.empty_like(mu)
    nv.check(lib.r2d2_target_smoothing(nv.dptr(mu), nv.dptr(out), n, 1.0, 0.3, 9, 0, 4, nv.current_stream()))
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    low = np.float32(np.float32(0.9) - np.float32(0.3))
    assert got.max() == 1.0 and got.min() == low and (got == low).sum() > 100 and (got == 1.0).sum() > 100
    want = t3.smooth(np.full(n, np.float32(0.9), np.float64), 1.0, float(np.float32(0.3)), 9, 0, 4)
    assert np.abs(got - want).max() < 1e-6


# ---------------------------------------------------------------------------------------------------- 4. float64
def _check(E, kw, actor, critic, batches, iters, extra, td=None, is_weight=None, probe_clip=False):
    cfg_kw = dict(kw, **extra)
    if probe_clip:
        eng0 = E.LearnerEngine(E.PathConfig(**kw, twin_critic=True))
        c2 = _np(eng0.views("critic2"))
        eng0.close()
        probe = t3.TD3Oracle(actor, critic, critic2=c2, twin=True, grad_clip=1e30, burn_in=kw["burn_in"],
                             learning=kw["learning"], n_step=kw["n_step"])
        probe.iteration(batches[0])
        cfg_kw["grad_clip_norm"] = float(np.float32(0.1 * min(probe.norms.values())))
    eng = E.LearnerEngine(E.PathConfig(**cfg_kw))
    eng.load_state_dicts(actor, critic)
    c2 = _np(eng.views("critic2"))
    c = eng.cfg
    ol = t3.TD3Oracle(actor, critic, critic2=c2, twin=True, sigma=float(np.float32(c.target_noise)),
                      noise_clip=float(np.float32(c.target_noise_clip)), seed=c.target_noise_seed,
                      target_tau=float(np.float32(c.target_tau)), grad_clip=c.grad_clip_norm, td=td,
                      burn_in=kw["burn_in"], learning=kw["learning"], n_step=kw["n_step"], target_interval=c.target_interval)
    errs = {}
    for it in range(iters):
        batch = dict(batches[it % len(batches)])
        if is_weight is not None:
            batch["is_weight"] = is_weight
        eng.set_batch(batch)
        eng.step()
        ref = ol.iteration(batch)
        torch.cuda.synchronize()
        for k, mine in (("q_value", eng.q_value), ("q_value2", eng.q_value2), ("target_q_value", eng.target_q_value),
                        ("priority", eng.priority)):
            errs[f"{k}/{it}"] = rel_l2(mine.cpu().numpy(), ref[k])
    for net in ("actor", "critic", "critic2", "target_actor", "target_critic", "target_critic2"):
        for k, v in eng.views(net).items():
            errs[f"{net}/{k}"] = rel_l2(v.cpu().numpy(), getattr(ol, net)[k])
    for net in ("actor", "critic", "critic2"):
        adam = getattr(ol, net + "_adam")
        for what, key in (("exp_avg", "m/"), ("exp_avg_sq", "v/")):
            for k, v in eng.views(net, what).items():
                errs[f"{what}/{net}/{k}"] = rel_l2(v.cpu().numpy(), adam[key + k])
    eng.close()
    bad = {k: v for k, v in errs.items() if not v < TOL}
    assert not bad, bad
    return max(errs.values())


SETTINGS = {"smooth": dict(TD3), "smooth_polyak_clip": dict(TD3, target_tau=0.005, target_interval=1)}


@pytest.mark.parametrize("setting", sorted(SETTINGS))
@pytest.mark.parametrize("name", ["ref_pend_h128.npz", "ref_walker_h128.npz"])
def test_runs_against_oracle_on_goldens(E, name, setting):
    g = load_golden(name)
    kw = dict(obs=int(g["cfg/obs_size"]), act=int(g["cfg/n_actions"]), hidden=int(g["cfg/hidden"]),
              batch=int(g["cfg/batch_size"]), burn_in=int(g["cfg/burn_in"]), learning=int(g["cfg/learning"]),
              n_step=int(g["cfg/n_step"]))
    n_it = len({k.split("/")[0] for k in g if k.startswith("it")})
    worst = _check(E, kw, golden_params(g, "init/actor"), golden_params(g, "init/critic"),
                   [golden_batch(g, i) for i in range(n_it)], 12, SETTINGS[setting],
                   probe_clip=setting == "smooth_polyak_clip")
    print(f"{name} {setting}: worst relative error {worst:.3e}")


def _port_run(E, kw, iters, extra, seed=1, n_batches=3, **check_kw):
    pc = ref_port.PathConfig(**kw)
    port = ref_port.PortLearner(pc, seed=seed)
    sd = lambda m: {k: v.detach().numpy() for k, v in m.state_dict().items()}  # noqa: E731
    return _check(E, kw, sd(port.actor), sd(port.critic),
                  [ref_port.synthetic_batch(pc, seed=6 + i) for i in range(n_batches)], iters, extra, **check_kw)


def test_runs_against_oracle_cfg2(E):
    kw = dict(obs=17, act=6, hidden=256, batch=256, burn_in=40, learning=80, n_step=5)
    print(f"cfg-2: worst relative error {_port_run(E, kw, 6, SETTINGS['smooth']):.3e}")


def test_rescaling_and_importance_weights_against_oracle(E):
    kw = dict(obs=11, act=3, hidden=128, batch=32, burn_in=10, learning=20, n_step=3)
    w = np.random.default_rng(3).uniform(0.2, 1.0, kw["batch"]).astype(np.float32)
    w[0] = 1.0
    extra = dict(TD3, value_rescaling="invertible", rescaling_eps=1e-3, is_exponent=0.6)
    worst = _port_run(E, kw, 6, extra, td=ro.td("invertible", float(np.float32(1e-3)), "squared", w.astype(np.float64)),
                      is_weight=w)
    print(f"invertible + IS weights: worst relative error {worst:.3e}")


@pytest.mark.parametrize("act", [1, 64])
def test_action_widths_through_the_smoothing_kernel(E, act):
    kw = dict(obs=7, act=act, hidden=64, batch=16, burn_in=4, learning=8, n_step=2)
    print(f"A={act}: worst relative error {_port_run(E, kw, 4, SETTINGS['smooth']):.3e}")


# ---------------------------------------------------------------------------------------------------- 5. schedules
SCHED = dict(TD3, target_tau=0.3, target_interval=3, grad_clip_norm=0.05)


def test_pipelined_step_matches_sequential_bit_for_bit(E):
    """Interval 3: on two of three iterations the next batch's target chains (and their noise) run ahead."""
    cfg = E.PathConfig(**SMALL, **SCHED)
    pc = ref_port.PathConfig(**SMALL)
    steps = 7
    batches = [ref_port.synthetic_batch(pc, seed=40 + it) for it in range(steps + 1)]
    seq = E.LearnerEngine(cfg, seed=3)
    seq_prio = []
    for it in range(steps):
        seq.set_batch(batches[it])
        seq.step()
        seq_prio.append(seq.priority.clone())
    pip = E.LearnerEngine(cfg, seed=3)
    pip_prio = []
    pip.set_batch(batches[0])
    for it in range(steps):
        def hook(eng, used, it=it):
            pip_prio.append(used.priority.clone())
            eng.set_batch(batches[it + 1])
        pip.step(prefetch=hook)
    torch.cuda.synchronize()
    for a, b in zip(seq_prio, pip_prio):
        assert torch.equal(a, b)
    _assert_same_bits(_snapshot(seq), _snapshot(pip))


def _replay_fed(E, steps):
    cfg = E.PathConfig(obs=11, act=3, hidden=128, batch=32, burn_in=10, learning=20, n_step=3, **SCHED)
    rng = np.random.default_rng(5)
    rp = E.DeviceReplay(cfg, capacity_rows=24 * (120 + cfg.n_step))
    rp.add_episodes([episode(rng, cfg, 120) for _ in range(24)])
    eng = E.LearnerEngine(cfg, seed=7)
    gen = torch.Generator(device="cuda").manual_seed(11)

    def hook(e, used):
        rp.update_priorities(used.leaf_idx, used.priority)
        rp.sample_into(e, generator=gen)

    rp.sample_into(eng, generator=gen)
    for _ in range(steps):
        eng.step(prefetch=hook)
    out = _snapshot(eng)
    rp.close()
    eng.close()
    return out


def test_replay_fed_runs_are_bitwise_reproducible(E):
    _assert_same_bits(_replay_fed(E, 7), _replay_fed(E, 7))


def test_resumed_run_is_bit_identical(E):
    cfg = E.PathConfig(**SMALL, **SCHED)
    pc = ref_port.PathConfig(**SMALL)
    a = E.LearnerEngine(cfg, seed=9)
    for it in range(2):
        a.set_batch(ref_port.synthetic_batch(pc, seed=it))
        a.step()
    st = a.training_state()
    assert {"critic2", "target_critic2", "critic2_optimizer"} <= set(st) and st["twin_critic"] is True
    b = E.LearnerEngine(cfg, seed=123)
    b.load_training_state(st)
    for it in range(2, 7):
        batch = ref_port.synthetic_batch(pc, seed=it)
        for e in (a, b):
            e.set_batch(batch)
            e.step()
    _assert_same_bits(_snapshot(a), _snapshot(b))
    a.close()
    b.close()


# ---------------------------------------------------------------------------------------------------- 6. data parallel
DP = dict(obs=6, act=2, hidden=64, batch=8, burn_in=4, learning=6, n_step=2, target_interval=2)


def test_dp_identical_shards_without_noise_give_the_single_engine_bits(E):
    pc = ref_port.PathConfig(**{k: v for k, v in DP.items() if k != "target_interval"})
    batches = [ref_port.synthetic_batch(pc, seed=60 + i) for i in range(4)]
    one = E.LearnerEngine(E.PathConfig(**DP, twin_critic=True), seed=2)
    for b in batches:
        one.set_batch(b)
        one.step()
    grp = PeerGroup(2, dict(DP, twin_critic=True), seed=2)
    grp.run([[b, b] for b in batches])
    grp.flush()
    grp.check_status()
    torch.cuda.synchronize()
    for r, eng in enumerate(grp.engines):
        for net in ("actor", "critic", "target_actor", "target_critic"):
            assert torch.equal(eng.flat[net], one.flat[net]), (r, net)
        for d in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(getattr(eng, d)["critic"], getattr(one, d)["critic"]), (r, d)
    grp.close()
    one.close()


def test_dp_disjoint_shards_with_rank_keyed_noise_against_oracle(E):
    kw = dict(DP, batch=16)
    pc = ref_port.PathConfig(**{k: v for k, v in kw.items() if k != "target_interval"})
    batches = [ref_port.synthetic_batch(pc, seed=80 + i) for i in range(5)]
    grp = PeerGroup(2, dict(kw, batch=kw["batch"] // 2, **TD3), seed=2)     # every rank one half of the global batch
    for r, eng in enumerate(grp.engines):
        eng.set_target_smoothing(rank=r)
    e0 = grp.engines[0]
    ol = t3.TD3Oracle(_np(e0.views("actor")), _np(e0.views("critic")), critic2=_np(e0.views("critic2")), twin=True,
                      sigma=float(np.float32(0.2)), noise_clip=0.5, burn_in=kw["burn_in"], learning=kw["learning"],
                      n_step=kw["n_step"], target_interval=kw["target_interval"])
    shards = [split_batch(b, 2) for b in batches]
    grp.run(shards)
    grp.flush()
    grp.check_status()
    for s in shards:
        ol.iteration(s)
    errs = {}
    for net in ("actor", "critic", "critic2", "target_actor", "target_critic", "target_critic2"):
        for k, v in e0.views(net).items():
            errs[f"{net}/{k}"] = rel_l2(v.cpu().numpy(), getattr(ol, net)[k])
    grp.close()
    bad = {k: v for k, v in errs.items() if not v < TOL}
    assert not bad, bad


# ---------------------------------------------------------------------------------------------------- 7. drop-in
def test_dropin_learner_with_td3(monkeypatch):
    import sys
    for k, v in dict(R2D2_OBS_SIZE="5", R2D2_N_ACTIONS="2", R2D2_HIDDEN="64", R2D2_BATCH="4", R2D2_TWIN_CRITIC="1",
                     R2D2_TARGET_NOISE="0.2", R2D2_TARGET_NOISE_CLIP="0.5", R2D2_TARGET_NOISE_SEED="3",
                     R2D2_TARGET_TAU="0.005", R2D2_TARGET_INTERVAL="1").items():
        monkeypatch.setenv(k, v)
    mods = ("actor", "learner", "replay_memory", "models", "utils")
    for m in mods:
        sys.modules.pop(m, None)
    import actor as dropin_actor
    import learner as dropin_learner
    with tempfile.TemporaryDirectory() as d:
        cwd = os.getcwd()
        os.chdir(d)
        try:
            os.makedirs("model_data")
            os.makedirs("memory_data")
            lr = dropin_learner.Learner(n_actors=2)
            c = lr.engine.cfg
            assert (c.twin_critic, c.target_noise, c.target_noise_clip, c.target_noise_seed) == (True, 0.2, 0.5, 3)
            for aid in range(2):
                a = dropin_actor.Actor(aid)
                a.env.episode_len = 150
                a.run(max_episodes=5)
            lr.model_save_interval = 2
            lr.memory_update_interval = 2
            lr.run(max_steps=4)
            torch.cuda.synchronize()
            assert lr.engine.step_count == 4
            assert np.isfinite(lr.engine.losses.cpu().numpy()).all() and len(lr.engine.losses) == 3
            md = torch.load(os.path.join("model_data", "model.pt"), map_location="cpu")
            assert sorted(md) == ["actor", "critic", "target_actor", "target_critic"]
            assert md["critic"]["l3.bias"].numel() == 2 and lr.engine.flat["critic"].numel() == 2 * lr.engine._critic2_off
            lr.update_target_model()
            assert torch.equal(lr.engine.flat["target_critic"], lr.engine.flat["critic"])
        finally:
            os.chdir(cwd)
            for m in mods:
                sys.modules.pop(m, None)


# ---------------------------------------------------------------------------------------------------- 8. two GPUs
def _dp_worker(rank, world, port, out_dir):
    import torch.distributed as dist
    from r2d2_b200 import engine
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(f"cuda:{rank}"))
    cfg = engine.PathConfig(**SMALL, **SCHED)
    eng = engine.LearnerEngine(cfg, device=f"cuda:{rank}", seed=5)
    eng.enable_data_parallel()
    rng = np.random.default_rng(100 + rank)
    rp = engine.DeviceReplay(cfg, capacity_rows=8000, device=f"cuda:{rank}")
    rp.add_episodes([episode(rng, cfg, int(rng.integers(30, 90))) for _ in range(30)])
    gen = torch.Generator(device=f"cuda:{rank}").manual_seed(7 + rank)

    def hook(e, used):
        rp.update_priorities(used.leaf_idx, used.priority)
        rp.sample_into(e, generator=gen)

    rp.sample_into(eng, generator=gen)
    for _ in range(4):
        eng.step(prefetch=hook)
    torch.cuda.synchronize()
    ok = bool(eng.replicas_identical()) and eng.peer_status() == 0 and eng._rank == rank
    np.save(os.path.join(out_dir, f"rank{rank}.npy"), np.array([ok]))
    dist.barrier()
    dist.destroy_process_group()


def test_two_gpu_replicas_stay_identical_with_td3():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    import torch.multiprocessing as mp
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_dp_worker, args=(2, 29700 + os.getpid() % 100, d), nprocs=2, join=True)
        for r in range(2):
            assert np.load(os.path.join(d, f"rank{r}.npy"))[0], f"rank {r}: replicas diverged"

"""Optimiser-step extras on the GPU: the Polyak target update fused into the Adam launches (target_tau) and per-net
global gradient-norm clipping (grad_clip_norm) - against torch's soft_update bit for bit, against the float64 oracle
over multi-iteration runs, the defaults against the plain path, and the pipelined / resumed / repeated schedules against
each other."""
import os
import tempfile
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from conftest import golden_batch, golden_params, load_golden, rel_l2
from oracle import ref_port
from optim_oracle import ClipHook, PolyakOracle
from test_gpu_prioritized_replay import episode

pytestmark = pytest.mark.gpu

TOL = 1e-3
SMALL = dict(obs=6, act=2, hidden=64, batch=8, burn_in=4, learning=6, n_step=2)


@pytest.fixture(scope="module")
def eng_mod():
    from r2d2_b200 import engine
    return engine


def _snapshot(eng):
    torch.cuda.synchronize()
    out = {f"flat.{n}": eng.flat[n].clone() for n in ("actor", "critic", "target_actor", "target_critic")}
    for d, name in ((eng.exp_avg, "m"), (eng.exp_avg_sq, "v")):
        out.update({f"{name}.{n}": d[n].clone() for n in ("actor", "critic")})
    out.update({k: getattr(eng, k).clone() for k in ("q_value", "target_q_value", "priority", "losses", "grad_norms")})
    return out


def _assert_same_bits(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert torch.equal(a[k], b[k]), k


# ---------------------------------------------------------------------------------------------------- 1. torch parity
def test_polyak_update_is_torch_soft_update_bit_for_bit(eng_mod):
    """One update iteration: each target equals utils.soft_update, run by torch on the same device tensors with the
    float32 value of tau, applied to the targets before the step and the post-step weights."""
    import utils
    tau = float(np.float32(0.005))
    cfg = eng_mod.PathConfig(**SMALL, target_tau=0.005, target_interval=1)
    eng = eng_mod.LearnerEngine(cfg, seed=2)
    g = torch.Generator().manual_seed(5)
    for n in ("target_actor", "target_critic"):                 # targets that differ from the nets
        eng.flat[n].add_(0.01 * torch.randn(eng.flat[n].shape, generator=g).to(eng.device))
    before = {n: eng.flat[n].clone() for n in ("target_actor", "target_critic")}
    eng.set_batch(ref_port.synthetic_batch(ref_port.PathConfig(**SMALL), seed=1))
    eng.step()
    torch.cuda.synchronize()
    for net in ("actor", "critic"):
        want = SimpleNamespace(parameters=lambda t=before["target_" + net]: [t])
        utils.soft_update(want, SimpleNamespace(parameters=lambda p=eng.flat[net]: [p]), tau)
        assert torch.equal(eng.flat["target_" + net], before["target_" + net]), net
        assert not torch.equal(eng.flat["target_" + net], eng.flat[net])


# ---------------------------------------------------------------------------------------------------- 2. float64 oracle
def _check_against_oracle(eng_mod, kw, actor, critic, batches, tau, interval, iters):
    probe = ClipHook(0.0)
    PolyakOracle(actor, critic, burn_in=kw["burn_in"], learning=kw["learning"], n_step=kw["n_step"]).iteration(
        batches[0], keep=False, grad_hook=probe)
    clip = float(np.float32(0.1 * min(probe.norms.values())))       # both nets clip on the first iteration
    cfg = eng_mod.PathConfig(**kw, target_tau=tau, target_interval=interval, grad_clip_norm=clip)
    eng = eng_mod.LearnerEngine(cfg)
    eng.load_state_dicts(actor, critic)
    ol = PolyakOracle(actor, critic, burn_in=kw["burn_in"], learning=kw["learning"], n_step=kw["n_step"],
                      target_interval=interval, target_tau=float(np.float32(tau)))
    hook = ClipHook(clip)
    errs, norm_errs, clipped = {}, {}, 0
    for it in range(iters):
        batch = batches[it % len(batches)]
        eng.set_batch(batch)
        eng.step()
        ref = ol.iteration(batch, grad_hook=hook)
        torch.cuda.synchronize()
        norms = eng.grad_norms.cpu().numpy()
        for i, net in enumerate(("critic", "actor")):
            # the kernel against float64 on the same gradient block, and against the oracle's norm, whose gradient
            # differs from the bf16x3 one by up to a few 1e-5 (DESIGN §3)
            own = np.sqrt(np.sum(np.square(eng.grads[net].cpu().numpy().astype(np.float64))))
            norm_errs[f"kernel/{net}/{it}"] = (abs(norms[i] / own - 1.0), 1e-6)
            norm_errs[f"oracle/{net}/{it}"] = (abs(norms[i] / hook.norms[net] - 1.0), 1e-4)
            clipped += hook.norms[net] > clip
        if it:                                               # later iterations see the updated weights and targets
            errs[f"q/{it}"] = rel_l2(eng.q_value.cpu().numpy(), ref["q_value"])
            errs[f"target/{it}"] = rel_l2(eng.target_q_value.cpu().numpy(), ref["target_q_value"])
            errs[f"prio/{it}"] = rel_l2(eng.priority.cpu().numpy(), ref["priority"])
    for net in ("actor", "critic"):
        for what, mine, theirs in (("params", eng.views(net), getattr(ol, net)),
                                   ("target", eng.views("target_" + net), getattr(ol, "target_" + net)),
                                   ("m", eng.views(net, "exp_avg"), {k: ol.__dict__[net + "_adam"]["m/" + k] for k in eng_mod.PARAM_KEYS}),
                                   ("v", eng.views(net, "exp_avg_sq"), {k: ol.__dict__[net + "_adam"]["v/" + k] for k in eng_mod.PARAM_KEYS})):
            for k in eng_mod.PARAM_KEYS:
                errs[f"{what}/{net}/{k}"] = rel_l2(mine[k].cpu().numpy(), theirs[k])
    assert clipped >= 2
    bad = {k: v for k, v in errs.items() if not v < TOL}
    assert not bad, bad
    bad = {k: v for k, (v, bar) in norm_errs.items() if not v < bar}
    assert not bad, bad
    eng.close()
    return max(errs.values())


@pytest.mark.parametrize("tau,interval", [(0.05, 1), (0.3, 3)])
@pytest.mark.parametrize("name", ["ref_pend_h128.npz", "ref_walker_h128.npz"])
def test_runs_against_oracle_on_goldens(eng_mod, name, tau, interval):
    g = load_golden(name)
    kw = dict(obs=int(g["cfg/obs_size"]), act=int(g["cfg/n_actions"]), hidden=int(g["cfg/hidden"]),
              batch=int(g["cfg/batch_size"]), burn_in=int(g["cfg/burn_in"]), learning=int(g["cfg/learning"]),
              n_step=int(g["cfg/n_step"]))
    n_it = len({k.split("/")[0] for k in g if k.startswith("it")})
    worst = _check_against_oracle(eng_mod, kw, golden_params(g, "init/actor"), golden_params(g, "init/critic"),
                                  [golden_batch(g, i) for i in range(n_it)], tau, interval, 12)
    print(f"{name} tau={tau} interval={interval}: worst relative error {worst:.3e}")


@pytest.mark.parametrize("tau,interval", [(0.05, 1), (0.3, 3)])
def test_runs_against_oracle_cfg2(eng_mod, tau, interval):
    kw = dict(obs=17, act=6, hidden=256, batch=256, burn_in=40, learning=80, n_step=5)
    pc = ref_port.PathConfig(**kw)
    port = ref_port.PortLearner(pc, seed=1)
    sd = lambda m: {k: v.detach().numpy() for k, v in m.state_dict().items()}  # noqa: E731
    worst = _check_against_oracle(eng_mod, kw, sd(port.actor), sd(port.critic),
                                  [ref_port.synthetic_batch(pc, seed=6 + i) for i in range(3)], tau, interval, 6)
    print(f"cfg-2 tau={tau} interval={interval}: worst relative error {worst:.3e}")


# ---------------------------------------------------------------------------------------------------- 3. defaults
def _fixed_batch_run(eng_mod, steps=4, **extra):
    cfg = eng_mod.PathConfig(**SMALL, target_interval=2, **extra)
    eng = eng_mod.LearnerEngine(cfg, seed=3)
    pc = ref_port.PathConfig(**SMALL)
    for it in range(steps):
        eng.set_batch(ref_port.synthetic_batch(pc, seed=20 + it))
        eng.step()
    out = _snapshot(eng)
    out["launches"] = eng.launches_per_iteration
    eng.close()
    return out


def test_clip_bound_that_never_clips_keeps_the_unclipped_bits(eng_mod):
    off, big = _fixed_batch_run(eng_mod), _fixed_batch_run(eng_mod, grad_clip_norm=1e30)
    assert big.pop("launches") == off.pop("launches") + 2           # one norm kernel per net
    norms = big.pop("grad_norms")
    assert (norms > 0).all() and torch.equal(off.pop("grad_norms"), torch.zeros_like(norms))   # off: nothing computed
    _assert_same_bits(off, big)


def test_default_launch_count_is_unchanged(eng_mod):
    base = _fixed_batch_run(eng_mod)["launches"]
    assert _fixed_batch_run(eng_mod, target_tau=1.0, grad_clip_norm=0.0)["launches"] == base
    assert _fixed_batch_run(eng_mod, target_tau=0.5)["launches"] == base          # the blend rides on the Adam launches
    assert _fixed_batch_run(eng_mod, grad_clip_norm=0.01)["launches"] == base + 2


def test_library_rejects_bad_values(eng_mod):
    eng = eng_mod.LearnerEngine(eng_mod.PathConfig(**SMALL))
    lib = eng.lib
    for tau in (0.0, -0.5, 1.0001, float("nan"), float("inf")):
        assert lib.r2d2_learner_set_target_tau(eng._h, tau) == -2                # R2D2_ERR_ARG
    for m in (-1.0, float("nan"), float("inf")):
        assert lib.r2d2_learner_set_grad_clip(eng._h, m) == -2
    assert lib.r2d2_learner_set_target_tau(eng._h, 1.0) == 0 and lib.r2d2_learner_set_grad_clip(eng._h, 0.0) == 0
    eng.close()


# ---------------------------------------------------------------------------------------------------- 4. schedules
def test_pipelined_step_matches_sequential_bit_for_bit(eng_mod):
    """At interval 1 every iteration updates the targets, so the pipelined step never runs the next target chains
    ahead and calls the hook at the end: the same kernels in the same order as the sequential loop."""
    cfg = eng_mod.PathConfig(**SMALL, target_tau=0.05, target_interval=1, grad_clip_norm=0.01)
    pc = ref_port.PathConfig(**SMALL)
    steps = 6
    batches = [ref_port.synthetic_batch(pc, seed=40 + it) for it in range(steps + 1)]
    seq = eng_mod.LearnerEngine(cfg, seed=3)
    seq_prio = []
    for it in range(steps):
        seq.set_batch(batches[it])
        seq.step()
        seq_prio.append(seq.priority.clone())
    pip = eng_mod.LearnerEngine(cfg, seed=3)
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
    a, b = _snapshot(seq), _snapshot(pip)
    _assert_same_bits(a, b)
    assert (a["grad_norms"] > 0.01).any()


def _replay_fed(eng_mod, steps):
    cfg = eng_mod.PathConfig(obs=11, act=3, hidden=128, batch=32, burn_in=10, learning=20, n_step=3,
                             target_tau=0.3, target_interval=3, grad_clip_norm=0.05)
    rng = np.random.default_rng(5)
    rp = eng_mod.DeviceReplay(cfg, capacity_rows=24 * (120 + cfg.n_step))
    rp.add_episodes([episode(rng, cfg, 120) for _ in range(24)])
    eng = eng_mod.LearnerEngine(cfg, seed=7)
    gen = torch.Generator(device="cuda").manual_seed(11)

    def hook(e, used):
        rp.update_priorities(used.leaf_idx, used.priority)
        rp.sample_into(e, generator=gen)

    rp.sample_into(eng, generator=gen)
    for _ in range(steps):
        eng.step(prefetch=hook)
    out = _snapshot(eng)
    rp.close()
    return out, eng


def test_replay_fed_runs_are_bitwise_reproducible(eng_mod):
    """Interval 3: the next batch's target chains run ahead on two of three iterations and wait on the third."""
    a, ea = _replay_fed(eng_mod, 7)
    b, eb = _replay_fed(eng_mod, 7)
    _assert_same_bits(a, b)
    assert not torch.equal(a["flat.target_critic"], a["flat.critic"])
    ea.close()
    eb.close()


def test_resumed_run_is_bit_identical(eng_mod):
    cfg = eng_mod.PathConfig(**SMALL, target_tau=0.3, target_interval=3, grad_clip_norm=0.05)
    pc = ref_port.PathConfig(**SMALL)
    a = eng_mod.LearnerEngine(cfg, seed=9)
    for it in range(2):
        a.set_batch(ref_port.synthetic_batch(pc, seed=it))
        a.step()
    st = a.training_state()
    b = eng_mod.LearnerEngine(cfg, seed=123)                   # different initial weights: everything comes from the state
    b.load_training_state(st)
    for it in range(2, 7):                                       # crosses the Polyak updates at steps 3 and 6
        batch = ref_port.synthetic_batch(pc, seed=it)
        for e in (a, b):
            e.set_batch(batch)
            e.step()
    _assert_same_bits(_snapshot(a), _snapshot(b))


# ---------------------------------------------------------------------------------------------------- 5. drop-in
def test_dropin_learner_with_soft_targets_and_clipping(monkeypatch):
    import sys
    for k, v in dict(R2D2_OBS_SIZE="5", R2D2_N_ACTIONS="2", R2D2_HIDDEN="64", R2D2_BATCH="4", R2D2_TARGET_TAU="0.05",
                     R2D2_TARGET_INTERVAL="1", R2D2_GRAD_CLIP="0.5").items():
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
            assert (c.target_tau, c.target_interval, c.grad_clip_norm) == (0.05, 1, 0.5)
            for aid in range(2):
                a = dropin_actor.Actor(aid)
                a.env.episode_len = 150
                a.run(max_episodes=5)
            lr.model_save_interval = 2
            lr.memory_update_interval = 2
            lr.run(max_steps=4)
            torch.cuda.synchronize()
            assert lr.engine.step_count == 4
            assert np.isfinite(lr.engine.losses.cpu().numpy()).all()
            norms = lr.engine.grad_norms.cpu().numpy()
            assert np.isfinite(norms).all() and (norms > 0).all()
            for net in ("actor", "critic"):                      # soft targets: neither the old nets nor a copy
                assert not torch.equal(lr.engine.flat["target_" + net], lr.engine.flat[net])
        finally:
            os.chdir(cwd)
            for m in mods:
                sys.modules.pop(m, None)


# ---------------------------------------------------------------------------------------------------- 6. two GPUs
def _dp_worker(rank, world, port, out_dir):
    import torch.distributed as dist
    from r2d2_b200 import engine
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(f"cuda:{rank}"))
    cfg = engine.PathConfig(**SMALL, target_tau=0.05, target_interval=1, grad_clip_norm=0.05)
    eng = engine.LearnerEngine(cfg, device=f"cuda:{rank}", seed=5)
    eng.enable_data_parallel()
    rng = np.random.default_rng(100 + rank)                                  # every rank its own shard
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
    ok = bool(eng.replicas_identical()) and eng.peer_status() == 0
    np.save(os.path.join(out_dir, f"rank{rank}.npy"), np.array([ok]))
    dist.barrier()
    dist.destroy_process_group()


def test_two_gpu_replicas_stay_identical_with_clipping_and_polyak():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    import torch.multiprocessing as mp
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_dp_worker, args=(2, 29800 + os.getpid() % 100, d), nprocs=2, join=True)
        for r in range(2):
            assert np.load(os.path.join(d, f"rank{r}.npy"))[0], f"rank {r}: replicas diverged"

"""Helpers shared by the learner tests: error bounds local to one action column, batch tile or unit group, the float64
oracle of a PathConfig and the one check of an engine against it, bit snapshots of an engine, replay episodes, draws
and fed runs, the schedule comparisons (pipelined, resumed), the drop-in learner on a fake engine (CPU) and trained for a few
steps (GPU), and the two-GPU NCCL replica check."""
import contextlib
import os
import socket
import sys
import tempfile

import numpy as np
import pytest

from conftest import golden_batch, golden_params, load_golden, rel_l2
from oracle import learner_oracle as lo
from oracle import ref_port

TOL = 1e-3
SMALL = dict(obs=6, act=2, hidden=64, batch=8, burn_in=4, learning=6, n_step=2)
REPLAY = dict(obs=11, act=3, hidden=128, batch=32, burn_in=10, learning=20, n_step=3)


def _f32(x):
    return float(np.float32(x))


def col_err(x, ref, A):
    """max over action columns j of ||x_j - ref_j|| / (||ref|| / sqrt(A)); both reshaped to [-1, A].  Normalised by the
    RMS column norm, so a column whose reference is near zero does not blow the ratio up; a relative L2 norm over a whole
    tensor would dilute an error confined to one column by about sqrt(A)."""
    x = np.asarray(x, np.float64).reshape(-1, A)
    ref = np.asarray(ref, np.float64).reshape(-1, A)
    rms_col = np.linalg.norm(ref) / np.sqrt(A)
    return float(np.linalg.norm(x - ref, axis=0).max() / max(rms_col, 1e-30))


def _worst_group(x, ref, axis, size):
    """max over consecutive groups of `size` indices along `axis` (the last group may be shorter) of the relative L2
    norm within the group."""
    x = np.moveaxis(np.asarray(x, np.float64), axis, 0)
    ref = np.moveaxis(np.asarray(ref, np.float64), axis, 0)
    worst = 0.0
    for g in range(0, x.shape[0], size):
        d, r = np.linalg.norm(x[g:g + size] - ref[g:g + size]), np.linalg.norm(ref[g:g + size])
        worst = max(worst, float(d / max(r, 1e-30)))
    return worst


def tile_err(x, ref, NB, axis=-2):
    """Worst relative L2 over the batch tiles of NB rows (one scan cluster each) along the batch axis, the ragged last
    tile counted on its own: a whole-tensor norm dilutes an error confined to one tile of B / NB by sqrt(B / NB)."""
    return _worst_group(x, ref, axis, NB)


def step_err(x, ref, axis=0):
    """Worst relative L2 over the single time rows along `axis`: a whole-tensor norm over T rows dilutes an error confined
    to one step by about sqrt(T).  A row is measured against its own reference norm, or against 1e-3 of the RMS row norm
    when its own is smaller (far from the head a BPTT row can decay below fp32's range, where float64 still has digits)."""
    x = np.moveaxis(np.asarray(x, np.float64), axis, 0).reshape(np.shape(x)[axis], -1)
    ref = np.moveaxis(np.asarray(ref, np.float64), axis, 0).reshape(x.shape)
    rn = np.linalg.norm(ref, axis=1)
    floor = 1e-3 * np.sqrt(np.mean(rn * rn))
    return float((np.linalg.norm(x - ref, axis=1) / np.maximum(np.maximum(rn, floor), 1e-30)).max())


def unit_group_err(x, ref, H, axis=-1):
    """Worst relative L2 over the groups of 32 hidden units (one cluster CTA each) along a unit axis of length H or 4H;
    on a 4H axis the groups are taken per gate block (i, f, g, o), so no group straddles two gates."""
    x, ref = np.asarray(x, np.float64), np.asarray(ref, np.float64)
    n = x.shape[axis]
    assert n in (H, 4 * H), f"unit axis of length {n} at H = {H}"
    if n == H:
        return _worst_group(x, ref, axis, 32)
    return max(_worst_group(np.take(x, range(q * H, (q + 1) * H), axis), np.take(ref, range(q * H, (q + 1) * H), axis),
                            axis, 32) for q in range(4))


# ------------------------------------------------------------------------------------------------ cases
def golden_case(name):
    """(PathConfig fields, actor, critic, batches) of a reference golden."""
    g = load_golden(name)
    kw = dict(obs=int(g["cfg/obs_size"]), act=int(g["cfg/n_actions"]), hidden=int(g["cfg/hidden"]),
              batch=int(g["cfg/batch_size"]), burn_in=int(g["cfg/burn_in"]), learning=int(g["cfg/learning"]),
              n_step=int(g["cfg/n_step"]))
    n_it = len({k.split("/")[0] for k in g if k.startswith("it")})
    return kw, golden_params(g, "init/actor"), golden_params(g, "init/critic"), [golden_batch(g, i) for i in range(n_it)]


def port_case(kw, seed=1, n_batches=3, batch_seed=6):
    """(actor, critic, batches): the reference port's initial nets and its synthetic batches."""
    pc = ref_port.PathConfig(**kw)
    port = ref_port.PortLearner(pc, seed=seed)
    sd = lambda m: {k: v.detach().numpy() for k, v in m.state_dict().items()}  # noqa: E731
    return sd(port.actor), sd(port.critic), [ref_port.synthetic_batch(pc, seed=batch_seed + i) for i in range(n_batches)]


def episode(rng, cfg, E, p_lo=0.01, zero_pad=False):
    """One actor episode of E rows plus n_step terminal pad rows, as DeviceReplay.add_episodes takes it; zero_pad: obs,
    act and rew of the pad rows zeroed (the same draws either way)."""
    n_rows = E + cfg.n_step
    term = np.zeros(n_rows, np.float32)
    term[E:] = 1
    obs = rng.standard_normal((n_rows, cfg.obs)).astype(np.float32)
    act = rng.uniform(-1, 1, (n_rows, cfg.act)).astype(np.float32)
    rew = rng.standard_normal(n_rows).astype(np.float32)
    if zero_pad:
        obs[E:], act[E:], rew[E:] = 0, 0, 0
    return (obs, act, rew, term, (0.1 * rng.standard_normal((E, 4, 2, cfg.hidden))).astype(np.float32),
            rng.uniform(p_lo, 1.0, E - (cfg.burn_in + cfg.learning)).astype(np.float32))


def gather_out(cfg, B):
    import torch
    T = cfg.rows
    return {"obs": torch.empty(T, B, cfg.obs, device="cuda"), "act": torch.empty(T, B, cfg.act, device="cuda"),
            "rew": torch.empty(T, B, device="cuda"), "term": torch.empty(T, B, device="cuda"),
            "states": torch.empty(4, 2, B, cfg.hidden, device="cuda")}


def draw(rp, cfg, kind, u=None, leaf=None, beta=0.6):
    """One draw of `kind` ("plain", "weighted", "chosen": r2d2_replay_gather at the given leaves) from DeviceReplay rp
    into fresh buffers, as host arrays: leaf, w (weighted), obs, act, rew, term, states."""
    import torch
    from r2d2_b200 import native as nv
    B = u.numel() if leaf is None else leaf.numel()
    out = gather_out(cfg, B)
    ptrs = [nv.dptr(out[k]) for k in ("obs", "act", "rew", "term", "states")]
    lib, s = nv.lib(), nv.current_stream()
    if kind == "chosen":
        nv.check(lib.r2d2_replay_gather(rp._h, nv.dptr(leaf, torch.int64), B, *ptrs, s))
        out["leaf"] = leaf.clone()
    else:
        out["leaf"] = torch.empty(B, dtype=torch.int64, device="cuda")
        if kind == "plain":
            nv.check(lib.r2d2_replay_sample(rp._h, nv.dptr(u), B, nv.dptr(out["leaf"], torch.int64), *ptrs, s))
        else:
            out["w"] = torch.empty(B, device="cuda")
            nv.check(lib.r2d2_replay_sample_weighted(rp._h, nv.dptr(u), B, float(beta), nv.dptr(out["leaf"], torch.int64),
                                                     nv.dptr(out["w"]), *ptrs, s))
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}


# ------------------------------------------------------------------------------------------------ float64 oracle
def oracle_for(cfg, actor, critic, critic2=None):
    """The float64 oracle learner of a PathConfig.  The library holds target_tau, rescaling_eps, target_noise and
    target_noise_clip in float32, so the oracle gets their float32 values."""
    return lo.OracleLearner(actor, critic, burn_in=cfg.burn_in, learning=cfg.learning, n_step=cfg.n_step,
                            target_interval=cfg.target_interval, target_tau=_f32(cfg.target_tau),
                            grad_clip=cfg.grad_clip_norm, value_rescaling=cfg.value_rescaling,
                            rescaling_eps=_f32(cfg.rescaling_eps), priority_metric=cfg.priority_metric,
                            twin=cfg.twin_critic, critic2=critic2, target_noise=_f32(cfg.target_noise),
                            target_noise_clip=_f32(cfg.target_noise_clip), target_noise_seed=cfg.target_noise_seed)


def _np(views):
    return {k: v.detach().cpu().numpy() for k, v in views.items()}


def check_against_oracle(E, cfg_kw, actor, critic, batches, iters, *, weights=None, first=0, probe_clip=False,
                         norms=False):
    """`iters` iterations of the engine of PathConfig(**cfg_kw) on batches[it % len(batches)] (with is_weight =
    weights(it) when given) against oracle_for of the same config.  Within TOL relative L2: q, target and priority (and
    q_value2 with the twin) of every iteration from `first` on; every trained net, its target and both Adam moments at the
    end.  probe_clip: clip at a tenth of the smaller first-iteration norm of the plain (twin) learner, so that every net
    clips from the first iteration on.  norms: grad_norms within 1e-6 of the float64 norm of the engine's own gradient
    block and within 1e-4 of the oracle's pre-clip norm, and at least two clipped norms.  Returns the worst relative
    error."""
    import torch
    twin = cfg_kw.get("twin_critic", False)
    if probe_clip:
        c2 = None
        if twin:                                      # critic 2 starts from the engine's own initial weights
            eng0 = E.LearnerEngine(E.PathConfig(**cfg_kw))
            c2 = _np(eng0.views("critic2"))
            eng0.close()
        probe = lo.OracleLearner(actor, critic, burn_in=cfg_kw["burn_in"], learning=cfg_kw["learning"],
                                 n_step=cfg_kw["n_step"], twin=twin, critic2=c2)
        probe.iteration(batches[0], keep=False)
        cfg_kw = dict(cfg_kw, grad_clip_norm=_f32(0.1 * min(probe.norms.values())))
    eng = E.LearnerEngine(E.PathConfig(**cfg_kw))
    eng.load_state_dicts(actor, critic)
    cfg = eng.cfg
    ol = oracle_for(cfg, actor, critic, _np(eng.views("critic2")) if twin else None)
    outputs = ("q_value", "q_value2", "target_q_value", "priority") if twin else ("q_value", "target_q_value", "priority")
    errs, norm_errs, clipped = {}, {}, 0
    for it in range(iters):
        batch = dict(batches[it % len(batches)])
        if weights is not None:
            batch["is_weight"] = weights(it)
        eng.set_batch(batch)
        eng.step()
        ref = ol.iteration(batch)
        torch.cuda.synchronize()
        if norms:
            got = eng.grad_norms.cpu().numpy()
            for i, net in enumerate(("critic", "actor")):
                # the kernel against float64 on the same gradient block, and against the oracle's norm, whose gradient
                # differs from the bf16x3 one by up to a few 1e-5 (DESIGN §3)
                own = np.sqrt(np.sum(np.square(eng.grads[net].cpu().numpy().astype(np.float64))))
                norm_errs[f"kernel/{net}/{it}"] = (abs(got[i] / own - 1.0), 1e-6)
                norm_errs[f"oracle/{net}/{it}"] = (abs(got[i] / ol.norms[net] - 1.0), 1e-4)
                clipped += ol.norms[net] > cfg.grad_clip_norm
        if it >= first:
            for k in outputs:
                errs[f"{k}/{it}"] = rel_l2(getattr(eng, k).cpu().numpy(), ref[k])
    nets = ("actor", "critic", "critic2") if twin else ("actor", "critic")
    for net in nets:
        adam = getattr(ol, net + "_adam")
        for what, mine, theirs in (("params", eng.views(net), getattr(ol, net)),
                                   ("target", eng.views("target_" + net), getattr(ol, "target_" + net)),
                                   ("m", eng.views(net, "exp_avg"), {k: adam["m/" + k] for k in lo.PARAM_KEYS}),
                                   ("v", eng.views(net, "exp_avg_sq"), {k: adam["v/" + k] for k in lo.PARAM_KEYS})):
            for k in lo.PARAM_KEYS:
                errs[f"{what}/{net}/{k}"] = rel_l2(mine[k].cpu().numpy(), theirs[k])
    eng.close()
    if norms:
        assert clipped >= 2
        bad = {k: v for k, (v, bar) in norm_errs.items() if not v < bar}
        assert not bad, bad
    bad = {k: v for k, v in errs.items() if not v < TOL}
    assert not bad, bad
    return max(errs.values())


# ------------------------------------------------------------------------------------------------ engine runs
def snapshot(eng):
    """Clones of everything an iteration leaves behind: nets, targets, Adam moments and the per-iteration outputs."""
    import torch
    torch.cuda.synchronize()
    out = {f"flat.{n}": eng.flat[n].clone() for n in ("actor", "critic", "target_actor", "target_critic")}
    for d, name in ((eng.exp_avg, "m"), (eng.exp_avg_sq, "v")):
        out.update({f"{name}.{n}": d[n].clone() for n in ("actor", "critic")})
    out.update({k: getattr(eng, k).clone() for k in ("q_value", "target_q_value", "priority", "losses", "grad_norms")})
    if eng.q_value2 is not None:
        out["q_value2"] = eng.q_value2.clone()
    return out


def assert_same_bits(a, b):
    import torch
    assert a.keys() == b.keys()
    for k in a:
        assert torch.equal(a[k], b[k]), k


def fixed_run(E, steps=4, setter=None, **extra):
    """snapshot() plus the launch count after `steps` sequential iterations of a seeded SMALL engine on synthetic
    batches, target interval 2; setter(engine) runs before the first step."""
    import torch
    eng = E.LearnerEngine(E.PathConfig(**SMALL, target_interval=2, **extra), seed=3)
    if setter:
        setter(eng)
    pc = ref_port.PathConfig(**SMALL)
    for it in range(steps):
        eng.set_batch(ref_port.synthetic_batch(pc, seed=20 + it))
        eng.step()
    out = snapshot(eng)
    out["launches"] = torch.tensor(eng.launches_per_iteration)
    eng.close()
    return out


def replay_fed_run(E, steps, seed=7, setup=None, beta=None, replay_cfg=None, keep=(), **extra):
    """snapshot() plus the launch count and the engine attributes named in `keep` after `steps` pipelined iterations of
    an engine of PathConfig(REPLAY updated by extra) fed from a seeded replay shard of 24 episodes (replay_cfg: the
    shard's own config, if it differs), each draw's priorities written back before the next (at `beta`, default the
    config's); setup(engine) runs before the first draw."""
    import torch
    cfg = E.PathConfig(**dict(REPLAY, **extra))
    rng = np.random.default_rng(5)
    rp = E.DeviceReplay(replay_cfg or cfg, capacity_rows=24 * (120 + cfg.n_step))
    rp.add_episodes([episode(rng, cfg, 120) for _ in range(24)])
    eng = E.LearnerEngine(cfg, seed=seed)
    if setup is not None:
        setup(eng)
    gen = torch.Generator(device="cuda").manual_seed(11)
    draw = {} if beta is None else {"beta": beta}

    def hook(e, used):
        rp.update_priorities(used.leaf_idx, used.priority)
        rp.sample_into(e, generator=gen, **draw)

    rp.sample_into(eng, generator=gen, **draw)
    for _ in range(steps):
        eng.step(prefetch=hook)
    out = snapshot(eng)
    out.update({k: getattr(eng, k).clone() for k in keep}, launches=torch.tensor(eng.launches_per_iteration))
    rp.close()
    eng.close()
    return out


def assert_pipelined_matches_sequential(E, cfg, steps):
    """The pipelined step drawing the next batch from its prefetch hook against the sequential loop on the same
    batches: every iteration's priorities and the final snapshot bit for bit.  Returns that snapshot."""
    import torch
    pc = ref_port.PathConfig(**{k: getattr(cfg, k) for k in SMALL})
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
    a, b = snapshot(seq), snapshot(pip)
    assert_same_bits(a, b)
    seq.close()
    pip.close()
    return a


def assert_resumed_run_is_bit_identical(E, cfg, check_state=None):
    """Two iterations, training_state(), a differently seeded engine loading it, then both on five more batches: the same
    bits.  check_state(state) runs on the saved state."""
    pc = ref_port.PathConfig(**{k: getattr(cfg, k) for k in SMALL})
    a = E.LearnerEngine(cfg, seed=9)
    for it in range(2):
        a.set_batch(ref_port.synthetic_batch(pc, seed=it))
        a.step()
    st = a.training_state()
    if check_state is not None:
        check_state(st)
    b = E.LearnerEngine(cfg, seed=123)                  # different initial weights: everything comes from the state
    b.load_training_state(st)
    for it in range(2, 7):
        batch = ref_port.synthetic_batch(pc, seed=it)
        for e in (a, b):
            e.set_batch(batch)
            e.step()
    assert_same_bits(snapshot(a), snapshot(b))
    a.close()
    b.close()


# ------------------------------------------------------------------------------------------------ drop-in learner
class _FakeEngine:
    def __init__(self, cfg, device=None):
        self.cfg, self.device = cfg, device

    def enable_data_parallel(self):
        pass

    def views(self, net):
        return {}


def fake_engine_learner(monkeypatch, tmp_path, **env):
    """The drop-in Learner built in tmp_path with the environment `env` on a stand-in engine that only keeps its
    PathConfig (no GPU needed)."""
    monkeypatch.setenv("R2D2_OBS_SIZE", "5")
    monkeypatch.setenv("R2D2_N_ACTIONS", "2")
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    from r2d2_b200 import engine
    monkeypatch.setattr(engine, "LearnerEngine", _FakeEngine)
    monkeypatch.chdir(tmp_path)
    os.makedirs("model_data", exist_ok=True)
    for m in ("learner", "replay_memory"):
        sys.modules.pop(m, None)
    import learner as dropin_learner
    try:
        return dropin_learner.Learner(n_actors=1)
    finally:
        for m in ("learner", "replay_memory"):
            sys.modules.pop(m, None)


@contextlib.contextmanager
def trained_dropin_learner(monkeypatch, **env):
    """The drop-in Learner (2 actors, hidden 64, batch 4, environment `env`) after two drop-in Actors wrote five 150-step
    episodes each and it ran four steps, in a temporary working directory: yields (learner, actors)."""
    import torch
    for k, v in dict(R2D2_OBS_SIZE="5", R2D2_N_ACTIONS="2", R2D2_HIDDEN="64", R2D2_BATCH="4", **env).items():
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
            actors = []
            for aid in range(2):
                a = dropin_actor.Actor(aid)
                a.env.episode_len = 150
                a.run(max_episodes=5)
                actors.append(a)
            lr.model_save_interval = 2
            lr.memory_update_interval = 2
            lr.run(max_steps=4)
            torch.cuda.synchronize()
            assert lr.engine.step_count == 4
            assert np.isfinite(lr.engine.losses.cpu().numpy()).all()
            yield lr, actors
        finally:
            os.chdir(cwd)
            for m in mods:
                sys.modules.pop(m, None)


# ------------------------------------------------------------------------------------------------ two GPUs
def _nccl_worker(rank, world, port, out_dir, cfg_kw):
    import torch
    import torch.distributed as dist
    from r2d2_b200 import engine
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(f"cuda:{rank}"))
    cfg = engine.PathConfig(**cfg_kw)
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
    ok = bool(eng.replicas_identical()) and eng.peer_status() == 0 and eng._rank == rank
    np.save(os.path.join(out_dir, f"rank{rank}.npy"), np.array([ok]))
    dist.barrier()
    dist.destroy_process_group()


def assert_two_gpu_replicas_stay_identical(cfg_kw):
    """Two NCCL ranks, each fed from its own replay shard for four pipelined steps, end with identical replicas."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    import torch.multiprocessing as mp
    with socket.socket() as s:                                               # a port nothing else holds
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_nccl_worker, args=(2, port, d, cfg_kw), nprocs=2, join=True)
        for r in range(2):
            assert np.load(os.path.join(d, f"rank{r}.npy"))[0], f"rank {r}: replicas diverged"

"""Learners trained on global sampling: replay-fed runs of LearnerEngine with PathConfig(global_sampling=True).

W = 1: the global mode's pipelined replay-fed run is the local mode's bit for bit (indices every iteration, nets, moments
and outputs at the end), and its write-back + draw cost a fixed 7 launches against the local 4 (3 unweighted).
W = 2, 4 in-process ranks (tests/global_harness.py), beta 0.6, alpha 0.9, pipelined and sequential, 6 iterations: every
draw restates from the device's written priorities, q / targets / priorities / nets stay within 1e-3 of the float64
learner on the global batch, pipelined equals sequential bit for bit, two seeded runs are identical, every status word
reads 0.  The drop-in Learner runs (twice) with R2D2_GLOBAL_SAMPLING=1; on >= 2 GPUs, two NCCL ranks keep identical
replicas and their draws restate."""
import os
import socket
import tempfile

import numpy as np
import pytest
import torch

from conftest import rel_l2
from global_harness import GlobalRun
from learner_harness import SMALL, assert_same_bits, episode, oracle_for, snapshot, trained_dropin_learner

pytestmark = pytest.mark.gpu

KW = dict(SMALL, hidden=64, priority_exponent=0.9, is_exponent=0.6, target_interval=3)
ITERS = 6


@pytest.fixture(scope="module")
def E():
    from r2d2_b200 import engine
    return engine


def _w1_run(E, global_sampling, steps=5):
    from r2d2_b200 import native as nv
    cfg = E.PathConfig(**dict(KW, global_sampling=global_sampling))
    rng = np.random.default_rng(5)
    rp = E.DeviceReplay(cfg, capacity_rows=4000)
    rp.add_episodes([episode(rng, cfg, int(rng.integers(30, 90))) for _ in range(24)])
    eng = E.LearnerEngine(cfg, seed=7)
    if global_sampling:
        rp.attach_group(eng)
    gen = torch.Generator(device="cuda").manual_seed(11)
    leaves, launches = [], []

    def hook(e, used):
        leaves.append(used.leaf_idx.clone())
        torch.cuda.synchronize()
        n0 = nv.lib().r2d2_launch_count()
        rp.update_priorities(used.leaf_idx, used.priority)
        rp.sample_into(e, generator=gen)
        launches.append(nv.lib().r2d2_launch_count() - n0)

    rp.sample_into(eng, generator=gen)
    for _ in range(steps):
        eng.step(prefetch=hook)
    out = snapshot(eng)
    out.update(leaf=torch.stack(leaves), tree=rp.tree_level(0).clone(), is_weight=eng.is_weight.clone())
    lpi = eng.launches_per_iteration
    status = rp.global_status()
    rp.close()
    eng.close()
    return out, launches, lpi, status


def test_w1_global_run_is_the_local_run_and_costs_seven_launches(E):
    loc, loc_launch, loc_lpi, _ = _w1_run(E, False)
    glo, glo_launch, glo_lpi, status = _w1_run(E, True)
    assert_same_bits(loc, glo)
    assert status == 0
    assert set(loc_launch) == {4}, loc_launch          # tree_sample, is_weight, gather, tree_update
    assert set(glo_launch) == {7}, glo_launch          # publish records, filtered update | root, draw, gather, deliver, receive
    assert loc_lpi == glo_lpi                          # the learner's phases do not change


def _parity(E, W, prefetch, seed=1):
    run = GlobalRun(E, W, KW, seed=seed)
    cfg = run.cfg
    L, A, B = cfg.learning, cfg.act, cfg.batch
    eng0 = run.g.engines[0]
    gcfg = E.PathConfig(**dict(KW, batch=W * B))
    actor = {k: v.cpu().numpy() for k, v in eng0.views("actor").items()}
    critic = {k: v.cpu().numpy() for k, v in eng0.views("critic").items()}
    ol = oracle_for(gcfg, actor, critic)
    errs = {}

    def on_critic(slot):
        batch = {k: run.slot_cat(k, slot).cpu().numpy() for k in ("obs", "act", "rew", "term", "is_weight")}
        st = run.slot_cat("states", slot).cpu().numpy()
        for i, k in enumerate(("a_state", "ta_state", "c_state", "tc_state")):
            batch[k] = st[i]
        ref = ol.iteration(batch)
        engs = run.g.engines
        cat = lambda xs: np.concatenate([x.reshape(L, -1, A) for x in xs], 1).reshape(-1, A)  # noqa: E731
        for k in ("q_value", "target_q_value"):
            e = rel_l2(cat([getattr(x, k).cpu().numpy() for x in engs]), ref[k])
            errs[k] = max(errs.get(k, 0.0), e)
        td = ref["average_td_loss"].reshape(-1, W * B)
        for r, x in enumerate(engs):      # learner.py:137's [b:-1:B] series over each rank's own columns
            f = td[:, r * B:(r + 1) * B].reshape(-1)
            want = np.asarray([0.9 * f[j:-1:B].max() + 0.1 * f[j:-1:B].mean() for j in range(B)])
            errs["priority"] = max(errs.get("priority", 0.0), rel_l2(x.priority.cpu().numpy(), want))

    try:
        run.run(ITERS, prefetch, on_critic=on_critic)
        assert run.status() == [0] * W
        run.g.check_status()
        for ref, got in run.draws:
            assert np.array_equal(ref[0], got[0]) and np.array_equal(ref[1], got[1])
        assert len(run.draws) == ITERS + (1 if prefetch else 0)
        shards = np.concatenate([got[0] for _, got in run.draws])
        assert len(set(shards.tolist())) == W, "some shard was never drawn from"
        for net in ("actor", "critic"):
            for what, mine, theirs in (("params", eng0.views(net), getattr(ol, net)),
                                       ("target", eng0.views("target_" + net), getattr(ol, "target_" + net))):
                for k, v in mine.items():
                    errs[f"{what}/{net}"] = max(errs.get(f"{what}/{net}", 0.0), rel_l2(v.cpu().numpy(), theirs[k]))
        snaps = [snapshot(e) for e in run.g.engines]
        for s in snaps[1:]:
            for k in ("flat.actor", "flat.critic", "m.actor", "v.critic"):
                assert torch.equal(s[k], snaps[0][k]), k
    finally:
        run.close()
    bad = {k: v for k, v in errs.items() if not v < 1e-3}
    assert not bad, bad
    return snaps[0], run.draws


@pytest.mark.parametrize("W", [2, 4])
def test_global_sampling_learners_against_float64(E, W):
    pip, pip_draws = _parity(E, W, True)
    seq, seq_draws = _parity(E, W, False)
    assert_same_bits(pip, seq)                                   # pipelined == sequential
    for (_, a), (_, b) in zip(pip_draws, seq_draws):
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    if W == 2:
        again, _ = _parity(E, W, True)
        assert_same_bits(pip, again)                             # two seeded runs are identical


def test_dropin_learner_runs_global_sampling(monkeypatch):
    with trained_dropin_learner(monkeypatch, R2D2_GLOBAL_SAMPLING="1") as (lr, _):
        assert lr.engine.cfg.global_sampling and lr.memory._dev.group is lr.engine
        lr.run(max_steps=2)                                      # a second run keeps the group
        torch.cuda.synchronize()
        assert lr.memory._dev.global_status() == 0
        assert np.isfinite(lr.engine.losses.cpu().numpy()).all()


# ------------------------------------------------------------------------------------------------ two GPUs
def _worker(rank, world, port, out_dir):
    import torch.distributed as dist
    from r2d2_b200 import engine
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(f"cuda:{rank}"))
    cfg = engine.PathConfig(**dict(KW, global_sampling=True))
    eng = engine.LearnerEngine(cfg, device=f"cuda:{rank}", seed=5)
    eng.enable_data_parallel()
    rng = np.random.default_rng(100 + rank)
    rp = engine.DeviceReplay(cfg, capacity_rows=8000, device=f"cuda:{rank}")
    rp.add_episodes([episode(rng, cfg, int(rng.integers(30, 90))) for _ in range(10 + 10 * rank)])
    rp.attach_group(eng)
    gen = torch.Generator(device=f"cuda:{rank}").manual_seed(7 + rank)
    rec = {}

    def record(i):
        torch.cuda.synchronize()
        rec[f"u{i}"] = eng.uniforms.cpu().numpy()
        rec[f"leaf{i}"] = eng.leaf_idx.cpu().numpy()
        rec[f"shard{i}"] = eng.shard_of(eng.leaf_idx).cpu().numpy()

    def levels(i):
        torch.cuda.synchronize()
        for l in range(rp.stats()["tree_levels"]):
            rec[f"lv{i}_{l}"] = rp.tree_level(l).cpu().numpy()

    levels(0)
    rp.sample_into(eng, generator=gen)
    record(0)
    for i in range(1, 5):                                       # sequential: levels between write-back and draw
        eng.step()
        rp.update_priorities(eng.leaf_idx, eng.priority)
        dist.barrier()
        levels(i)
        dist.barrier()
        rp.sample_into(eng, generator=gen)
        record(i)
    torch.cuda.synchronize()
    rec["ok"] = np.array([bool(eng.replicas_identical()) and eng.peer_status() == 0 and rp.global_status() == 0])
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), **rec)
    dist.barrier()
    dist.destroy_process_group()


def test_two_gpu_global_sampling_keeps_replicas_and_restates():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    import torch.multiprocessing as mp
    from oracle import global_sumtree as gs
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_worker, args=(2, port, d), nprocs=2, join=True)
        recs = [dict(np.load(os.path.join(d, f"rank{r}.npz"))) for r in range(2)]
    assert all(r["ok"][0] for r in recs)
    for i in range(5):
        lv = [[rec[k] for k in sorted((k for k in rec if k.startswith(f"lv{i}_")), key=lambda k: int(k.split("_")[1]))]
              for rec in recs]
        shard, leaf, _ = gs.global_draw(lv, np.concatenate([rec[f"u{i}"] for rec in recs]))
        assert np.array_equal(shard, np.concatenate([rec[f"shard{i}"] for rec in recs]))
        assert np.array_equal(leaf, np.concatenate([rec[f"leaf{i}"] for rec in recs]))

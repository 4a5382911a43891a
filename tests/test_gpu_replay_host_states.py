"""Recurrent states in pinned host memory (replay_state_memory="host", R2D2_REPLAY_HOST_GB) on the GPU.  The gather only
moves where the states are read from, so every check is bit for bit against the host model of the ring or against a
device-state shard fed the same operations:

1. seeded ingest / write-back / restore sequences on a host-state and a device-state shard side by side, each checked
   against oracle/replay_model.py after every operation, with every restore crossing tiers;
2. every state route (H = 8, 12, 13, 512) at the ring's last rows, add_episode's zero-filled state rows, the fp16
   overflow refusal, and an ingest issued on the stream right behind a draw;
3. snapshots between the tiers, both directions, same and other capacity, fp32 <-> fp16;
4. global sampling with one host-state and one device-state shard;
5. the replay-fed pipelined learner, and the drop-in Learner training, snapshotting and resuming with the variable set."""
import dataclasses
import os
import shutil
import sys

import numpy as np
import pytest
import torch

from learner_harness import assert_same_bits, draw, episode, golden_case, snapshot
from oracle.replay_model import ReplayModel
from test_gpu_replay_model import CAPACITIES, KW, U, WRITE_BACKS, check_against_model, ring_length, shard_episode
from r2d2_b200 import engine as E
from r2d2_b200 import native as nv

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _needs_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")


def tier(cfg, memory):
    return dataclasses.replace(cfg, replay_state_memory=memory)


def shard(cfg, memory, cap, max_sequences=0, eps=()):
    rp = E.DeviceReplay(tier(cfg, memory), capacity_rows=cap, max_sequences=max_sequences)
    if eps:
        rp.add_episodes(list(eps))
    return rp


def levels(rp):
    return [rp.tree_level(l).cpu().numpy().copy() for l in range(int(rp.stats()["tree_levels"]))]


def assert_draws_equal(a, b, where=""):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k].dtype == b[k].dtype and a[k].tobytes() == b[k].tobytes(), f"{where} {k}"


def assert_shards_equal(h, d, cfg, where=""):
    """Counters, FIFO table, every tree level, both draws at U and a gather at every live start: the same bits."""
    assert h.stats() == d.stats(), where
    assert h.snapshot_info() == d.snapshot_info(), where
    for a, b in zip(h.episodes(), d.episodes()):
        assert np.array_equal(a, b), where
    for l, (a, b) in enumerate(zip(levels(h), levels(d))):
        assert a.tobytes() == b.tobytes(), f"{where} level {l}"
    if not h.stats()["n_episodes"]:
        return
    u = torch.as_tensor(U).cuda()
    for kind in ("plain", "weighted"):
        assert_draws_equal(draw(h, cfg, kind, u), draw(d, cfg, kind, u), f"{where} {kind}")
    rs, nr, ns, _ = h.episodes()
    starts = np.concatenate([np.arange(s, s + n) for s, n in zip(rs, ns)] or [np.zeros(0, np.int64)])
    if starts.size:
        leaf = torch.as_tensor(starts[:4096]).cuda()
        assert_draws_equal(draw(h, cfg, "chosen", leaf=leaf), draw(d, cfg, "chosen", leaf=leaf), f"{where} chosen")


def host_bytes_of(cfg, cap):
    return cap * 8 * cfg.hidden * (2 if cfg.replay_state_dtype == "float16" else 4)


# ------------------------------------------------------------------------------------------------ 1. the model
@pytest.mark.parametrize("max_sequences", [0, "cap/3"])
@pytest.mark.parametrize("dtype", ["float32", "float16"])
@pytest.mark.parametrize("alpha", [1.0, 0.6])
@pytest.mark.parametrize("cap", CAPACITIES)
def test_random_sequence_against_model_and_device_tier(cap, alpha, dtype, max_sequences, tmp_path):
    cfg = E.PathConfig(**KW, priority_exponent=alpha, replay_state_dtype=dtype)
    W = cfg.rows
    ms = cap // 3 if max_sequences else 0
    rng = np.random.default_rng([cap, int(alpha * 10), int(dtype == "float16"), ms, 7])
    h, d = shard(cfg, "host", cap, ms), shard(cfg, "device", cap, ms)
    assert h.host_bytes() == host_bytes_of(cfg, cap) and d.host_bytes() == 0
    assert d.device_bytes() - h.device_bytes() == host_bytes_of(cfg, cap)
    m = ReplayModel.for_config(cfg, cap, ms)
    ops = ["file"] * 8 + ["wider"] * 4 + ["single"] * 3 + ["write-back"] * 5 + ["restore", "restore-other"]
    rng.shuffle(ops)
    ops = ["wider"] + ops
    n_wb = 0
    for i, op in enumerate(ops):
        where = f"op {i} ({op})"
        if op in ("file", "wider"):
            k = int(rng.integers(1, 7) if op == "file" else rng.integers(2, 7))
            if op == "file":
                lens = [ring_length(rng, m.capacity, W) for _ in range(k)]
            else:
                lo = max(W, m.capacity // k + 1)
                lens = [int(n) for n in rng.integers(lo, min(m.capacity, 2 * lo) + 1, k)]
            eps = [shard_episode(rng, cfg, n) for n in lens]
            want = m.add_episodes(eps)
            assert h.add_episodes(eps) == want and d.add_episodes(eps) == want, where
        elif op == "single":
            ep = shard_episode(rng, cfg, ring_length(rng, m.capacity, W))
            h.add_episode(*ep)
            d.add_episode(*ep)
            m.add_episode(*ep)
        elif op == "write-back":
            live = m.live_starts()
            if live.size == 0:
                continue
            n = WRITE_BACKS[n_wb % len(WRITE_BACKS)]
            n_wb += 1
            leaf = rng.choice(live, n)
            prio = rng.uniform(0.01, 2.0, n).astype(np.float32)
            prio[rng.random(n) < 0.1] = 0
            for rp in (h, d):
                rp.update_priorities(torch.as_tensor(leaf).cuda(), torch.as_tensor(prio).cuda())
            m.update_priorities(leaf, prio)
        else:                                      # each tier restores the other tier's file
            new_cap = m.capacity
            if op == "restore-other":
                new_cap = max(W, 2 * m.capacity // 3) if rng.random() < 0.5 else m.capacity + m.capacity // 3 + 1
            h.save_snapshot(str(tmp_path / f"h{i}"))
            d.save_snapshot(str(tmp_path / f"d{i}"))
            h.close()
            d.close()
            h, d = shard(cfg, "host", new_cap, ms), shard(cfg, "device", new_cap, ms)
            out_h = h.load_snapshot(str(tmp_path / f"d{i}"), restore_rng=False)
            out_d = d.load_snapshot(str(tmp_path / f"h{i}"), restore_rng=False)
            m, dropped = m.restored(new_cap)
            assert out_h["dropped"] == out_d["dropped"] == dropped, where
        try:
            check_against_model(h, m, cfg, beta=(0.6, 1.0)[i % 2])
            assert_shards_equal(h, d, cfg, where)
        except AssertionError as e:
            raise AssertionError(f"{where}: {e}") from e
    h.close()
    d.close()


# ------------------------------------------------------------------------------------------------ 2. edges
def _gather_states_only(rp, leaf):
    """r2d2_replay_gather with every output but the states NULL: only the state rows of `leaf` are read."""
    c = rp.cfg
    st = torch.empty(4, 2, leaf.numel(), c.hidden, device="cuda")
    nv.check(rp.lib.r2d2_replay_gather(rp._h, nv.dptr(leaf, torch.int64), leaf.numel(), None, None, None, None,
                                       nv.dptr(st), nv.current_stream()))
    torch.cuda.synchronize()
    return st.cpu().numpy()


@pytest.mark.parametrize("dtype", ["float32", "float16"])
@pytest.mark.parametrize("H", [8, 12, 13, 512])
def test_every_state_route_at_the_ring_end_and_zero_filled_rows(H, dtype):
    """H = 8 / 12 / 13 take the 16-byte, 8-byte and scalar routes of fp16 storage (16-byte / scalar of fp32), and 512
    the widest request.  The ring is filled to its last row with states on every row; add_episode then wraps with fewer
    state rows than rows, and those rows must read back as zeros in both tiers."""
    cfg = E.PathConfig(obs=5, act=3, hidden=H, batch=8, burn_in=2, learning=3, n_step=2, replay_state_dtype=dtype)
    T, cap = cfg.rows, 400
    rng = np.random.default_rng(H)
    h, d = shard(cfg, "host", cap), shard(cfg, "device", cap)
    for n in (100, 100, 100, 100):                 # exactly to the last row, states on every row
        ep = episode(rng, cfg, n - cfg.n_step)
        full = (0.5 * rng.standard_normal((n, 4, 2, H))).astype(np.float32)
        for rp in (h, d):
            rp.add_episode(ep[0], ep[1], ep[2], ep[3], full, ep[5])
    last = torch.arange(cap - 64, cap, dtype=torch.int64, device="cuda")
    a, b = _gather_states_only(h, last), _gather_states_only(d, last)
    assert a.tobytes() == b.tobytes() and np.abs(a).sum() > 0
    leaf = torch.arange(cap - T - 40, cap - T + 1, dtype=torch.int64, device="cuda")
    assert_draws_equal(draw(h, cfg, "chosen", leaf=leaf), draw(d, cfg, "chosen", leaf=leaf), "ring end")
    ep = episode(rng, cfg, 60)                      # 60 state rows of 62: wraps to row 0, evicts the first episode
    for rp in (h, d):
        rp.add_episode(*ep)
    assert h.episodes()[0][-1] == 0
    pad = torch.arange(58, 62, dtype=torch.int64, device="cuda")
    z = _gather_states_only(h, pad)
    assert z[:, :, 2:].tobytes() == np.zeros_like(z[:, :, 2:]).tobytes() and np.abs(z[:, :, :2]).sum() > 0
    assert z.tobytes() == _gather_states_only(d, pad).tobytes()
    assert_shards_equal(h, d, cfg, "after the wrap")
    h.close()
    d.close()


def test_fp16_overflow_refusal_leaves_both_tiers_untouched():
    cfg = E.PathConfig(obs=5, act=2, hidden=16, batch=8, burn_in=4, learning=6, n_step=2, replay_state_dtype="float16")
    rng = np.random.default_rng(9)
    eps = [episode(rng, cfg, int(rng.integers(cfg.rows + 20, cfg.rows + 60))) for _ in range(6)]
    h, d = shard(cfg, "host", 600, eps=eps), shard(cfg, "device", 600, eps=eps)
    u = torch.as_tensor(U).cuda()
    before = draw(h, cfg, "plain", u), levels(h)
    for bad in (65520.0, -1e30):
        big = [episode(rng, cfg, int(rng.integers(cfg.rows + 100, cfg.rows + 140))) for _ in range(3)]
        big[-1][4][-1, 3, 1, 5] = bad
        for rp in (h, d):
            with pytest.raises(nv.NativeError, match="65520"):
                rp.add_episodes(big)
            with pytest.raises(nv.NativeError, match="65520"):
                rp.add_episode(*big[-1])
        assert_shards_equal(h, d, cfg, f"after refusing {bad}")
        assert_draws_equal(before[0], draw(h, cfg, "plain", u))
        for a, b in zip(before[1], levels(h)):
            assert a.tobytes() == b.tobytes()
    h.close()
    d.close()


def test_ingest_right_behind_a_draw_on_the_same_stream():
    """A draw, then at once - no host synchronisation - a file wider than the ring that overwrites every row the draw
    reads: the drawn batch is the one taken with a synchronisation in between."""
    cfg = E.PathConfig(obs=17, act=6, hidden=512, batch=1024, burn_in=8, learning=16, n_step=3)
    rng = np.random.default_rng(21)
    eps = [episode(rng, cfg, 200) for _ in range(8)]
    cap = sum(e[0].shape[0] for e in eps)
    wider = [episode(rng, cfg, 300) for _ in range(6)]
    u = torch.rand(cfg.batch, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    got = {}
    for synced in (True, False):
        rp = shard(cfg, "host", cap, eps=eps)
        torch.cuda.synchronize()
        out = {k: torch.empty(cfg.rows, cfg.batch, n, device="cuda") for k, n in (("obs", cfg.obs), ("act", cfg.act))}
        out["states"] = torch.empty(4, 2, cfg.batch, cfg.hidden, device="cuda")
        leaf = torch.empty(cfg.batch, dtype=torch.int64, device="cuda")
        nv.check(rp.lib.r2d2_replay_sample(rp._h, nv.dptr(u), cfg.batch, nv.dptr(leaf, torch.int64), nv.dptr(out["obs"]),
                                           nv.dptr(out["act"]), None, None, nv.dptr(out["states"]), nv.current_stream()))
        if synced:
            torch.cuda.synchronize()
        rp.add_episodes(wider)
        torch.cuda.synchronize()
        got[synced] = {k: v.cpu().numpy() for k, v in out.items()}
        got[synced]["leaf"] = leaf.cpu().numpy()
        assert rp.stats()["n_episodes"] < len(wider)
        rp.close()
    assert_draws_equal(got[True], got[False])


# ------------------------------------------------------------------------------------------------ 3. snapshots
SNAP_KW = dict(obs=11, act=3, hidden=64, batch=16, burn_in=10, learning=20, n_step=3)


def _filled(cfg, memory, cap, seed=3):
    rng = np.random.default_rng(seed)
    rp = shard(cfg, memory, cap)
    gen = torch.Generator(device="cuda").manual_seed(seed)
    for _ in range(6):
        rp.add_episodes([episode(rng, cfg, int(rng.integers(cfg.rows + 10, cfg.rows + 110))) for _ in range(5)])
        leaf = rp.sample_indices(torch.rand(40, device="cuda", generator=gen))
        rp.update_priorities(leaf, torch.rand(40, device="cuda", generator=gen) * 3)
    torch.cuda.synchronize()
    return rp


@pytest.mark.parametrize("src_dtype, dst_dtype", [("float32", "float32"), ("float16", "float16"),
                                                  ("float32", "float16"), ("float16", "float32")])
@pytest.mark.parametrize("src_mem, dst_mem", [("host", "device"), ("device", "host")])
def test_snapshots_cross_tiers(src_mem, dst_mem, src_dtype, dst_dtype, tmp_path):
    """A file written by one tier, restored into the other at the same and at another capacity, equals the restore of
    the same file into a shard of the restoring tier's opposite - every row, leaf, level and draw."""
    cap = 3000
    src = _filled(E.PathConfig(**SNAP_KW, replay_state_dtype=src_dtype), src_mem, cap)
    path = str(tmp_path / "shard")
    src.save_snapshot(path)
    cfg = E.PathConfig(**SNAP_KW, replay_state_dtype=dst_dtype)
    for new_cap in (cap, cap // 2, 2 * cap):
        a, b = shard(cfg, dst_mem, new_cap), shard(cfg, src_mem, new_cap)
        oa, ob = a.load_snapshot(path, restore_rng=False), b.load_snapshot(path, restore_rng=False)
        assert oa["dropped"] == ob["dropped"]
        assert_shards_equal(a, b, cfg, f"capacity {new_cap}")
        a.close()
        b.close()
    src.close()


# ------------------------------------------------------------------------------------------------ 4. global sampling
class _Tiers:
    """Stands in for the engine module in GlobalRun: its shards get the tiers in `memories`, rank by rank."""

    def __init__(self, memories):
        self.memories = list(memories)

    def DeviceReplay(self, cfg, **kw):
        return E.DeviceReplay(tier(cfg, self.memories.pop(0)), **kw)


def test_global_sampling_w2_mixed_tiers():
    from global_harness import GlobalRun
    kw = dict(obs=7, act=3, hidden=32, batch=16, burn_in=4, learning=6, n_step=2)
    out = {}
    for memories in (("device", "device"), ("host", "device"), ("device", "host")):
        run = GlobalRun(_Tiers(memories), 2, kw)
        assert [rp.host_bytes() > 0 for rp in run.shards] == [m == "host" for m in memories]
        slots = []

        def on_critic(slot, run=run, slots=slots):
            slots.append({k: run.slot_cat(k, slot).cpu().numpy() for k in
                          ("obs", "act", "rew", "term", "states", "leaf_idx", "shard", "is_weight")})

        run.run(4, prefetch=True, on_critic=on_critic)
        assert run.status() == [0, 0]
        for ref, got in run.draws:
            assert np.array_equal(ref[0], got[0]) and np.array_equal(ref[1], got[1])
        torch.cuda.synchronize()
        out[memories] = (run.draws, slots, [snapshot(e) for e in run.g.engines],
                         [{k: run.slot_cat(k, s).cpu().numpy() for k in ("states", "leaf_idx", "is_weight")}
                          for s in (0, 1)])
        run.close()
    ref = out[("device", "device")]
    for memories in (("host", "device"), ("device", "host")):
        got = out[memories]
        assert len(got[0]) == len(ref[0]) and len(got[1]) == len(ref[1])
        for (_, a), (_, b) in zip(ref[0], got[0]):
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
        for a, b in zip(ref[1] + ref[3], got[1] + got[3]):
            assert_draws_equal(a, b, str(memories))
        for a, b in zip(ref[2], got[2]):
            assert_same_bits(a, b)


# ------------------------------------------------------------------------------------------------ 5. learner
def _fed_run(kw, memory, steps=6, seed=7):
    """snapshot() after `steps` pipelined replay-fed iterations, each draw's priorities written back before the next."""
    cfg = E.PathConfig(**kw)
    rng = np.random.default_rng(5)
    eps = [episode(rng, cfg, cfg.burn_in + cfg.learning + 60) for _ in range(max(12, cfg.batch // 8))]
    rp = shard(cfg, memory, sum(e[0].shape[0] for e in eps), eps=eps)
    eng = E.LearnerEngine(cfg, seed=seed)
    gen = torch.Generator(device="cuda").manual_seed(11)

    def hook(e, used):
        rp.update_priorities(used.leaf_idx, used.priority)
        rp.sample_into(e, generator=gen)

    rp.sample_into(eng, generator=gen)
    for _ in range(steps):
        eng.step(prefetch=hook)
    out = snapshot(eng)
    out["launches"] = torch.tensor(eng.launches_per_iteration)
    rp.close()
    eng.close()
    return out


@pytest.mark.parametrize("shapes", ["cfg2", "ref_walker_h128", "cfg2-fp16-per"])
def test_replay_fed_learner_host_equals_device(shapes):
    if shapes.startswith("cfg2"):
        kw = dict(obs=17, act=6, hidden=256, batch=256, burn_in=40, learning=80, n_step=5)
        if shapes.endswith("per"):
            kw.update(replay_state_dtype="float16", priority_exponent=0.6, is_exponent=0.4)
    else:
        kw = {k: v for k, v in golden_case(shapes + ".npz")[0].items() if k in E.PathConfig.__dataclass_fields__}
    assert_same_bits(_fed_run(kw, "device"), _fed_run(kw, "host"))


def test_dropin_learner_with_host_states_trains_snapshots_and_resumes(monkeypatch, tmp_path):
    """R2D2_REPLAY_HOST_GB set: the drop-in Learner trains, writes replay snapshots, and a run resumed from one
    continues bit for bit as the uninterrupted run.  (A resume onto the other tier restores the same rows, section 3,
    but at the default ring size of that tier, so its leaf indices - and draws - differ.)"""
    env = dict(R2D2_OBS_SIZE="5", R2D2_N_ACTIONS="2", R2D2_HIDDEN="64", R2D2_BATCH="4",
               R2D2_REPLAY_SNAPSHOT_INTERVAL="50", R2D2_REPLAY_HOST_GB="0.25")
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    monkeypatch.delenv("R2D2_RESUME", raising=False)
    mods = ("actor", "learner", "replay_memory", "models", "utils")
    for m in mods:
        sys.modules.pop(m, None)
    import actor as dropin_actor
    import learner as dropin_learner
    cwd = os.getcwd()
    files = tmp_path / "actor_files"

    def enter(name):
        d = tmp_path / name
        for sub in ("model_data", "memory_data"):
            (d / sub).mkdir(parents=True, exist_ok=True)
        os.chdir(d)

    def done(lr):
        torch.cuda.synchronize()
        out = {f"flat.{n}": lr.engine.flat[n].clone() for n in ("actor", "critic", "target_actor", "target_critic")}
        out.update({f"m.{n}": lr.engine.exp_avg[n].clone() for n in ("actor", "critic")})
        out.update({f"v.{n}": lr.engine.exp_avg_sq[n].clone() for n in ("actor", "critic")})
        out["step"] = torch.tensor(lr.engine.step_count)
        lr.engine.close()
        lr.memory.clear()
        return out

    def fed_run(name, steps):
        enter(name)
        for f in files.iterdir():
            shutil.copy(f, "memory_data")
        torch.cuda.manual_seed(1234)
        lr = dropin_learner.Learner(n_actors=2)
        lr.run(max_steps=steps)
        return lr

    try:
        enter("actors")
        lr = dropin_learner.Learner(n_actors=2)
        for aid in range(2):
            a = dropin_actor.Actor(aid)
            a.env.episode_len = 150
            a.run(max_episodes=5)
        shutil.copytree("memory_data", files)
        lr.engine.close()

        whole = fed_run("whole", 150)
        assert whole.memory._dev.host_bytes() == whole.memory._dev.stats()["capacity_rows"] * 8 * 64 * 4 > 0
        whole = done(whole)
        first = fed_run("resumed", 100)
        root = tmp_path / "resumed" / "model_data" / "replay_snapshot"
        assert sorted(os.listdir(root)) == ["step100"]
        done(first)
        monkeypatch.setenv("R2D2_RESUME", "1")
        lr = dropin_learner.Learner(n_actors=2)
        assert lr.engine.step_count == 100 and lr.memory._dev.host_bytes() > 0
        lr.run(max_steps=50)
        assert_same_bits(whole, done(lr))
    finally:
        os.chdir(cwd)
        for m in mods:
            sys.modules.pop(m, None)

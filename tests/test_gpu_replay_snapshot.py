"""Replay snapshots on the GPU: a save and restore into a fresh shard of the same capacity gives back every tree level,
every live row, the counters, decode and the LearnerReplayMemory mirror; an engine and replay that restore a snapshot
continue bit for bit as the run that wrote it (both state types, alpha / beta on, global sampling at W = 1); a change of
state type converts exactly or refuses an fp16 overflow; another capacity compacts the episodes as an ingest of the
survivors would place them; the drop-in Learner resumes from its newest complete snapshot as if it had not stopped."""
import os
import shutil
import sys
from ctypes import c_void_p

import numpy as np
import pytest

from learner_harness import assert_same_bits, episode, snapshot

pytestmark = pytest.mark.gpu

KW = dict(obs=11, act=3, hidden=64, batch=16, burn_in=10, learning=20, n_step=3, target_interval=4)


@pytest.fixture(scope="module")
def E():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from r2d2_b200 import engine
    return engine


def _p(a):
    return a.ctypes.data_as(c_void_p)


def live_rows(rp):
    """Every live episode's rows and leaves, FIFO order, in the stored types."""
    from r2d2_b200 import native as nv
    c = rp.cfg
    half = rp.snapshot_info()["state_storage"] == nv.STATE_F16
    out = {k: [] for k in ("obs", "act", "rew", "term", "states", "leaves")}
    for s, n in zip(*rp.episodes()[:2]):
        n = int(n)
        a = dict(obs=np.empty((n, c.obs), np.float32), act=np.empty((n, c.act), np.float32), rew=np.empty(n, np.float32),
                 term=np.empty(n, np.float32), states=np.empty((n, 4, 2, c.hidden), np.float16 if half else np.float32),
                 leaves=np.empty(n, np.float32))
        nv.check(rp.lib.r2d2_replay_export_rows(rp._h, int(s), n, *[_p(a[k]) for k in out], nv.current_stream()))
        for k in out:
            out[k].append(a[k])
    return {k: np.concatenate(v) if v else np.zeros(0) for k, v in out.items()}


def assert_rows_equal(a, b, keys=("obs", "act", "rew", "term", "states", "leaves")):
    for k in keys:
        assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape and a[k].tobytes() == b[k].tobytes(), k


def levels(rp):
    return [rp.tree_level(l).clone() for l in range(int(rp.stats()["tree_levels"]))]


def assert_levels_equal(a, b):
    la, lb = levels(a), levels(b)
    assert len(la) == len(lb)
    for l, (x, y) in enumerate(zip(la, lb)):
        assert x.equal(y), l


def gather(rp, leaf):
    import torch
    from r2d2_b200 import native as nv
    c, B = rp.cfg, leaf.numel()
    out = dict(obs=torch.empty(c.rows, B, c.obs, device="cuda"), act=torch.empty(c.rows, B, c.act, device="cuda"),
               rew=torch.empty(c.rows, B, device="cuda"), term=torch.empty(c.rows, B, device="cuda"),
               states=torch.empty(4, 2, B, c.hidden, device="cuda"))
    nv.check(rp.lib.r2d2_replay_gather(rp._h, nv.dptr(leaf, torch.int64), B, *[nv.dptr(out[k]) for k in
                                                                                 ("obs", "act", "rew", "term", "states")],
                                       nv.current_stream()))
    torch.cuda.synchronize()
    return out


def filled_shard(E, cfg, cap, n_files=6, seed=3, states=None):
    """A shard of capacity `cap` fed n_files files of 5 episodes, with random priority write-backs after each: it has
    wrapped, left a tail gap and evicted."""
    import torch
    rng = np.random.default_rng(seed)
    rp = E.DeviceReplay(cfg, capacity_rows=cap)
    gen = torch.Generator(device="cuda").manual_seed(seed)
    for f in range(n_files):
        eps = [episode(rng, cfg, int(rng.integers(cfg.rows + 10, cfg.rows + 110))) for _ in range(5)]
        if states is not None and f == n_files - 1:
            eps[-1][4][3, 2, 1, 5] = states
        rp.add_episodes(eps)
        leaf = rp.sample_indices(torch.rand(40, device="cuda", generator=gen))
        rp.update_priorities(leaf, torch.rand(40, device="cuda", generator=gen) * 3)
    torch.cuda.synchronize()
    info = rp.snapshot_info()
    rs = rp.episodes()[0]
    assert info["evicted_total"] > 0 and (np.diff(rs) < 0).any() and info["rows_used"] < cap
    return rp


# ------------------------------------------------------------------------------------------------ 1. round trip
@pytest.mark.parametrize("dtype, hidden", [("float32", 32), ("float16", 32), ("float16", 36)])
def test_round_trip_same_capacity(E, tmp_path, dtype, hidden):
    import torch
    from replay_memory import LearnerReplayMemory
    rng = np.random.default_rng(1)
    kw = dict(memory_sequence_size=4000, batch_size=8, obs_size=7, n_actions=2, hidden=hidden, capacity_rows=1500,
              priority_exponent=0.9, state_dtype=dtype)
    m = LearnerReplayMemory(**kw)
    for _ in range(28):
        Ep = int(rng.integers(70, 160))
        rows = [(rng.standard_normal(7).astype(np.float32), rng.uniform(-1, 1, 2).astype(np.float32),
                 [float(rng.standard_normal())], [1.0 if i >= Ep else 0.0]) for i in range(Ep + 5)]
        st = (0.3 * rng.standard_normal((Ep, 4, 2, hidden))).astype(np.float32)
        m.add_episode(rows, st, rng.uniform(0.01, 1, Ep - 60).astype(np.float32))
        leaf = m._dev.sample_indices(torch.rand(12, device="cuda"))
        m._dev.update_priorities(leaf, torch.rand(12, device="cuda") * 2)
    info = m._dev.snapshot_info()
    assert info["evicted_total"] > 0 and (np.diff(m._dev.episodes()[0]) < 0).any() and info["rows_used"] < 1500
    path = str(tmp_path / "shard")
    rng_state = torch.cuda.get_rng_state()
    m.save_snapshot(path, stage_bytes=37 * 4 * 8 * hidden)          # many chunks, one across the ring's wrap
    torch.rand(5, device="cuda")                                      # move the generator on
    m2 = LearnerReplayMemory(**kw)
    hdr = m2.load_snapshot(path)
    assert hdr["dropped"] == 0 and torch.cuda.get_rng_state().equal(rng_state)
    assert_levels_equal(m._dev, m2._dev)
    assert_rows_equal(live_rows(m._dev), live_rows(m2._dev))
    assert m2._dev.stats() == m._dev.stats() and m2._dev.snapshot_info() == info
    all_rows = np.arange(1500)
    for x, y in zip(m._dev.decode(all_rows), m2._dev.decode(all_rows)):
        assert np.array_equal(x, y)
    assert list(m2._episodes) == list(m._episodes) and m2.sequence_counter == m.sequence_counter
    assert len(m2.priority) == len(m.priority)
    for e in range(len(m.priority)):
        assert list(m2.priority[e]) == list(m.priority[e])
    torch.cuda.set_rng_state(rng_state)
    a = m.sample()
    torch.cuda.set_rng_state(rng_state)
    b = m2.sample()
    assert a[0] == b[0] and a[1] == b[1]
    for x, y in zip(a[2:], b[2:]):
        assert x.equal(y)
    m.clear()
    m2.clear()


# ------------------------------------------------------------------------------------------------ 2. continuation
def _attach_w1(eng, rp):
    import torch
    lay = eng.global_layout(1)
    buf = torch.zeros(int(lay.bytes) // 4, dtype=torch.float32, device="cuda")
    eng.use_global_slots(buf, lay)
    eng.global_peer_ptrs, eng._rank = [buf.data_ptr()], 0
    rp.attach_group(eng)
    return buf


@pytest.mark.parametrize("dtype, alpha, beta, global_sampling", [("float32", 1.0, 0.0, False),
                                                                 ("float16", 0.9, 0.6, False),
                                                                 ("float32", 0.9, 0.6, True),
                                                                 ("float16", 1.0, 0.0, True)])
def test_restored_run_continues_bit_for_bit(E, tmp_path, dtype, alpha, beta, global_sampling):
    import torch
    cfg = E.PathConfig(**KW, priority_exponent=alpha, is_exponent=beta, replay_state_dtype=dtype,
                       global_sampling=global_sampling)
    rng = np.random.default_rng(5)
    files = [[episode(rng, cfg, int(rng.integers(40, 120))) for _ in range(4)] for _ in range(8)]
    keep = []

    def make(seed):
        eng, rp = E.LearnerEngine(cfg, seed=seed), E.DeviceReplay(cfg, capacity_rows=1800, max_sequences=900)
        if global_sampling:
            keep.append(_attach_w1(eng, rp))
        return eng, rp

    def run(eng, rp, first, last, out):
        for t in range(first, last):
            rp.sample_into(eng)
            eng.step()
            rp.update_priorities(eng.leaf_idx, eng.priority)
            out.append((eng.leaf_idx.clone(), eng.priority.clone()))
            if (t + 1) % 3 == 0:
                rp.add_episodes(files[2 + (t + 1) // 3])

    torch.cuda.manual_seed(17)
    a, rpa = make(3)
    rpa.add_episodes(files[0] + files[1])
    run(a, rpa, 0, 6, [])
    st = a.training_state()
    path = str(tmp_path / "shard")
    rpa.save_snapshot(path, learner_step=6, stage_bytes=1 << 16)
    tail_a = []
    run(a, rpa, 6, 15, tail_a)
    b, rpb = make(99)                                  # other weights: everything comes from the state and the file
    b.load_training_state(st)
    assert rpb.load_snapshot(path)["learner_step"] == 6
    tail_b = []
    run(b, rpb, 6, 15, tail_b)
    torch.cuda.synchronize()
    for (la, pa), (lb, pb) in zip(tail_a, tail_b):
        assert la.equal(lb) and pa.equal(pb)
    assert_same_bits(snapshot(a), snapshot(b))
    assert_levels_equal(rpa, rpb)
    for x in (rpa, rpb, a, b):
        x.close()


# ------------------------------------------------------------------------------------------------ 3. state type
def test_fp16_snapshot_into_fp32_ring_gathers_the_same_bits(E, tmp_path):
    import torch
    c16 = E.PathConfig(**KW, replay_state_dtype="float16")
    src = filled_shard(E, c16, 2500)
    path = str(tmp_path / "s")
    src.save_snapshot(path)
    dst = E.DeviceReplay(E.PathConfig(**KW), capacity_rows=2500)
    dst.load_snapshot(path)
    assert_levels_equal(src, dst)
    leaf = src.sample_indices(torch.rand(300, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1)))
    a, b = gather(src, leaf), gather(dst, leaf)
    for k in a:
        assert a[k].equal(b[k]), k
    assert live_rows(dst)["states"].tobytes() == live_rows(src)["states"].astype(np.float32).tobytes()
    src.close()
    dst.close()


def test_fp32_snapshot_into_fp16_ring_rounds_as_ingest_does(E, tmp_path):
    import torch
    src = filled_shard(E, E.PathConfig(**KW), 2500)
    path = str(tmp_path / "s")
    src.save_snapshot(path)
    dst = E.DeviceReplay(E.PathConfig(**KW, replay_state_dtype="float16"), capacity_rows=2500)
    dst.load_snapshot(path)
    assert_levels_equal(src, dst)
    leaf = src.sample_indices(torch.rand(300, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2)))
    a, b = gather(src, leaf), gather(dst, leaf)
    for k in ("obs", "act", "rew", "term"):
        assert a[k].equal(b[k]), k
    assert b["states"].equal(a["states"].half().float())
    src.close()
    dst.close()


def _assert_empty(rp):
    info = rp.snapshot_info()
    assert all(info[k] == 0 for k in ("n_episodes", "head", "sequence_counter", "next_serial", "evicted_total",
                                      "rows_used")), info
    assert rp.stats()["total_priority"] == 0.0
    for lv in levels(rp):
        assert not lv.any()


def test_fp16_overflow_refuses_the_whole_restore(E, tmp_path):
    from r2d2_b200 import native as nv
    src = filled_shard(E, E.PathConfig(**KW), 2500, states=65520.0)
    path = str(tmp_path / "s")
    src.save_snapshot(path, stage_bytes=1 << 16)
    dst = E.DeviceReplay(E.PathConfig(**KW, replay_state_dtype="float16"), capacity_rows=2500)
    with pytest.raises(nv.NativeError, match="65520"):
        dst.load_snapshot(path)
    _assert_empty(dst)
    ok = filled_shard(E, E.PathConfig(**KW), 2500, seed=4)         # the emptied shard takes a good snapshot afterwards
    ok.save_snapshot(path)
    dst.load_snapshot(path)
    assert_levels_equal(ok, dst)
    for x in (src, dst, ok):
        x.close()


def test_bad_leaves_and_short_files_refuse_the_restore(E, tmp_path):
    from r2d2_b200 import native as nv
    from r2d2_b200 import replay_snapshot as rsnap
    src = filled_shard(E, E.PathConfig(**KW), 2500)
    path = str(tmp_path / "s")
    h = src.save_snapshot(path)
    raw = bytearray(open(path, "rb").read())
    rows0 = h.header_bytes + h.n_episodes * 24
    leaves0 = rows0 + rsnap._chunk_layout(h, min(h.chunk_rows, h.rows_used))[5][0]
    n_starts0 = int(src.episodes()[2][0])
    for row, value in ((0, np.float32(np.nan)), (1, np.float32(-1.0)), (2, np.float32(np.inf)),
                       (n_starts0, np.float32(0.5))):                  # the last: a row that starts no sequence
        bad = bytearray(raw)
        bad[leaves0 + 4 * row:leaves0 + 4 * row + 4] = value.tobytes()
        p = str(tmp_path / "bad")
        open(p, "wb").write(bad)
        dst = E.DeviceReplay(E.PathConfig(**KW), capacity_rows=2500)
        with pytest.raises(nv.NativeError, match="leaf"):
            dst.load_snapshot(p)
        _assert_empty(dst)
        dst.close()
    p = str(tmp_path / "short")
    open(p, "wb").write(raw[:-100])
    dst = E.DeviceReplay(E.PathConfig(**KW), capacity_rows=2500)
    with pytest.raises(ValueError, match="truncated"):
        dst.load_snapshot(p)
    _assert_empty(dst)
    dst.close()
    src.close()


# ------------------------------------------------------------------------------------------------ 4. capacity
def test_other_capacity_compacts_like_an_ingest_of_the_survivors(E, tmp_path):
    cfg = E.PathConfig(**KW)
    src = filled_shard(E, cfg, 3000, n_files=8)
    path = str(tmp_path / "s")
    src.save_snapshot(path, stage_bytes=1 << 16)
    info = src.snapshot_info()
    rs, nr, ns, _ = src.episodes()
    rows = live_rows(src)
    off = np.concatenate([[0], np.cumsum(nr)])
    for cap in (7001, int(info["rows_used"]) // 2 + 17):
        keep = len(nr)
        while nr[len(nr) - keep:].sum() > cap:
            keep -= 1
        gone = list(range(len(nr) - keep))
        dst = E.DeviceReplay(cfg, capacity_rows=cap)
        assert dst.load_snapshot(path)["dropped"] == len(gone)
        ref = E.DeviceReplay(cfg, capacity_rows=cap)
        ref.add_episodes([(rows["obs"][off[e]:off[e + 1]], rows["act"][off[e]:off[e + 1]], rows["rew"][off[e]:off[e + 1]],
                           rows["term"][off[e]:off[e + 1]], rows["states"][off[e]:off[e + 1]],
                           rows["leaves"][off[e]:off[e] + ns[e]]) for e in range(len(gone), len(nr))])
        assert_levels_equal(dst, ref)
        assert_rows_equal(live_rows(dst), live_rows(ref))
        assert np.array_equal(dst.episodes()[0], ref.episodes()[0])
        got = dst.snapshot_info()
        assert got["sequence_counter"] == info["sequence_counter"] - sum(int(nr[e]) - (cfg.burn_in + cfg.learning)
                                                                         for e in gone)
        assert got["evicted_total"] == info["evicted_total"] + len(gone)
        assert got["head"] == got["rows_used"] == int(nr[len(gone):].sum())
        assert got["next_serial"] == info["next_serial"]
        dst.close()
        ref.close()
    src.close()


# ------------------------------------------------------------------------------------------------ 5. drop-in Learner
def test_dropin_learner_resumes_from_its_newest_complete_snapshot(E, monkeypatch, tmp_path):
    import torch
    env = dict(R2D2_OBS_SIZE="5", R2D2_N_ACTIONS="2", R2D2_HIDDEN="64", R2D2_BATCH="4",
               R2D2_REPLAY_SNAPSHOT_INTERVAL="50")
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
        return d

    def done(lr):
        torch.cuda.synchronize()
        out = {f"flat.{n}": lr.engine.flat[n].clone() for n in ("actor", "critic", "target_actor", "target_critic")}
        out.update({f"m.{n}": lr.engine.exp_avg[n].clone() for n in ("actor", "critic")})
        out.update({f"v.{n}": lr.engine.exp_avg_sq[n].clone() for n in ("actor", "critic")})
        out["leaves"] = lr.memory._dev.tree_level(0).clone()
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
        enter("actors")                                     # two actor files, fed to every run below
        lr = dropin_learner.Learner(n_actors=2)
        for aid in range(2):
            a = dropin_actor.Actor(aid)
            a.env.episode_len = 150
            a.run(max_episodes=5)
        shutil.copytree("memory_data", files)
        lr.engine.close()

        whole = done(fed_run("whole", 150))
        first = fed_run("resumed", 100)
        root = tmp_path / "resumed" / "model_data" / "replay_snapshot"
        assert sorted(os.listdir(root)) == ["step100"]      # step50 went once step100 was complete
        assert sorted(os.listdir(root / "step100")) == ["COMPLETE", "learner_state.pt", "shard0of1"]
        done(first)
        # a newer snapshot that never completed (its marker missing, its shard cut short) is ignored
        shutil.copytree(root / "step100", root / "step150")
        os.remove(root / "step150" / "COMPLETE")
        with open(root / "step150" / "shard0of1", "r+b") as f:
            f.truncate(1000)
        torch.save({"bogus": True}, "model_data/learner_state.pt")   # newer than the snapshot: not what resumes
        monkeypatch.setenv("R2D2_RESUME", "1")
        lr = dropin_learner.Learner(n_actors=2)
        assert lr.engine.step_count == 100
        assert lr.memory.sequence_counter >= lr.batch_size * 100

        def no_wait(_):
            raise AssertionError("the warm-up gate waited after the restore")
        monkeypatch.setattr(dropin_learner, "sleep", no_wait)
        lr.run(max_steps=50)
        resumed = done(lr)
        assert sorted(os.listdir(root)) == ["step150"] and (root / "step150" / "COMPLETE").is_file()
        assert_same_bits(whole, resumed)
    finally:
        os.chdir(cwd)
        for m in mods:
            sys.modules.pop(m, None)

"""fp16 recurrent-state storage of the replay shard (r2d2_replay_options.state_storage = R2D2_STATE_F16) on the device.

The states are rounded once at ingest and widened exactly by the gather, so an fp16 shard must hand out exactly what an
fp32 shard hands out with its states rounded to fp16 (numpy's round-to-nearest-even): the same leaves, the same obs /
act / rew / term bits and np.float16-rounded states, on every gather route (H % 8 == 0, H % 4 == 0, odd H) and for the
plain, weighted, caller-chosen and global draws.  Bookkeeping (FIFO, ring wrap, the reference's counter) is the fp32
shard's; a value fp16 would overflow refuses the whole call and leaves the shard untouched; training on the rounded
states stays within 1e-3 of the float64 oracle and of the fp32-storage run."""
from ctypes import c_void_p

import numpy as np
import pytest
import torch

from conftest import rel_l2
from learner_harness import (REPLAY, TOL, assert_same_bits, check_against_oracle, draw, episode, golden_case,
                             port_case, snapshot)
from r2d2_b200 import engine as E
from r2d2_b200 import native as nv

pytestmark = pytest.mark.gpu

F16_EDGES = np.float32([2.0 ** -14, 2.0 ** -24, 2.0 ** -25, 2.0 ** -26, 3e-8, 1e-6, 1e-9, -1e-6, -0.0, 0.0, 65504.0,
                        -65504.0, 65519.99, -65519.99, 65505.0, np.nan, np.inf, -np.inf, 1.0 + 2.0 ** -11,
                        1.0 + 3 * 2.0 ** -11, 0.1, -0.7])


def f16(x):
    return np.asarray(x, np.float32).astype(np.float16).astype(np.float32)


def assert_rounded(got, src):
    """got == np.float16(src) widened to fp32, bit for bit; NaN compared by isnan."""
    got = np.asarray(got, np.float32)
    want = f16(src)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan)
    assert np.array_equal(got[~nan].view(np.uint32), want[~nan].view(np.uint32))


def lstm_like_states(rng, n, H):
    """[n,4,2,H]: h in (-1, 1), c a few units - what the four nets' cells hold."""
    s = np.empty((n, 4, 2, H), np.float32)
    s[:, :, 0] = np.tanh(rng.standard_normal((n, 4, H)))
    s[:, :, 1] = 2.0 * rng.standard_normal((n, 4, H))
    return s


def episodes_with_edges(rng, cfg, n_eps, lo=None, hi=None):
    lo, hi = lo or cfg.rows + 4, hi or cfg.rows + 40
    eps = []
    for _ in range(n_eps):
        ep = list(episode(rng, cfg, int(rng.integers(lo, hi))))
        st = lstm_like_states(rng, ep[4].shape[0], cfg.hidden)
        flat = st.reshape(-1)
        pos = rng.choice(flat.size, size=min(flat.size, 8 * F16_EDGES.size), replace=False)
        flat[pos] = np.resize(F16_EDGES, pos.size)
        ep[4] = st
        eps.append(tuple(ep))
    return eps


def shard(cfg, dtype, cap, eps=()):
    rp = E.DeviceReplay(E.PathConfig(**dict(cfg.__dict__, replay_state_dtype=dtype)), capacity_rows=cap)
    if eps:
        rp.add_episodes(list(eps))
    return rp


def assert_fp16_draw_is_rounded_fp32_draw(a32, a16):
    for k in a32:
        if k != "states":
            assert np.array_equal(a32[k], a16[k]), k
    assert_rounded(a16["states"], a32["states"])


# ------------------------------------------------------------------------------------------------ 1. bit-exact gather
@pytest.mark.parametrize("H", [512, 36, 33])
@pytest.mark.parametrize("kind", ["plain", "weighted", "chosen"])
def test_gather_is_the_rounded_fp32_gather(H, kind):
    """H = 512: 16-byte route, 36: 8-byte route, 33: scalar route.  The fp32 shard stores the originals, so its gather
    is the host rows; the fp16 shard's is the same with the states rounded."""
    cfg = E.PathConfig(obs=7, act=3, hidden=H, batch=64, burn_in=3, learning=5, n_step=2)
    rng = np.random.default_rng(H)
    eps = episodes_with_edges(rng, cfg, 10)
    cap = sum(e[0].shape[0] for e in eps) + 64
    s32, s16 = shard(cfg, "float32", cap, eps), shard(cfg, "float16", cap, eps)
    gen = torch.Generator(device="cuda").manual_seed(H)
    for _ in range(3):
        u = torch.rand(257, device="cuda", generator=gen)
        u[0] = 1.0 - 2.0 ** -24
        leaf = None
        if kind == "chosen":
            rows = s32.stats()["n_rows_used"]
            leaf = torch.randint(0, rows - cfg.rows, (257,), device="cuda", generator=gen)
        a32, a16 = draw(s32, cfg, kind, u, leaf), draw(s16, cfg, kind, u, leaf)
        assert_fp16_draw_is_rounded_fp32_draw(a32, a16)
        # and the fp32 gather is the host data: the start row's stored states, in net order
        ep_i, seq_i = s32.decode(a32["leaf"])
        for b in range(0, 257, 16):
            st = eps[ep_i[b]][4]
            src = st[seq_i[b]] if seq_i[b] < st.shape[0] else np.zeros((4, 2, H), np.float32)
            assert_rounded(a16["states"][:, :, b], src)
    s32.close()
    s16.close()


def test_sample_into_is_the_rounded_fp32_batch():
    cfg = E.PathConfig(**REPLAY)
    rng = np.random.default_rng(4)
    eps = episodes_with_edges(rng, cfg, 12, cfg.rows + 20, cfg.rows + 80)
    cap = sum(e[0].shape[0] for e in eps)
    s32, s16 = shard(cfg, "float32", cap, eps), shard(cfg, "float16", cap, eps)
    e32, e16 = E.LearnerEngine(cfg), E.LearnerEngine(cfg)
    u = torch.rand(cfg.batch, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    s32.sample_into(e32, u=u)
    s16.sample_into(e16, u=u)
    torch.cuda.synchronize()
    for k in ("leaf_idx", "obs", "act", "rew", "term"):
        assert torch.equal(getattr(e32, k), getattr(e16, k)), k
    assert_rounded(e16.states.cpu().numpy(), e32.states.cpu().numpy())
    for x in (e32, e16, s32, s16):
        x.close()


# ------------------------------------------------------------------------------------------------ 2. bookkeeping
def test_ingest_matches_reference_load_sequence_fp16(tmp_path, monkeypatch):
    """The reference's file sequence (tests/golden/ref_ingest.npz) through the drop-in LearnerReplayMemory in fp16
    mode: the reference's sequence counter and survivors after every file."""
    import os
    import sys
    from collections import deque

    from conftest import load_golden
    from oracle.make_golden import ingest_file_sequence
    g = load_golden("ref_ingest.npz")
    monkeypatch.chdir(tmp_path)
    os.makedirs("memory_data")
    sys.modules.pop("replay_memory", None)
    import replay_memory as dropin_rm
    mem = dropin_rm.LearnerReplayMemory(memory_sequence_size=int(g["memory_sequence_size"]), batch_size=4,
                                        obs_size=4, n_actions=2, hidden=8, capacity_rows=4096, state_dtype="float16")
    for i, (actor_id, eps) in enumerate(ingest_file_sequence()):
        torch.save({"replay_memory": deque([e[0] for e in eps]), "recurrent_state": deque([e[1] for e in eps]),
                    "priority": deque([e[2] for e in eps]), "total_priority": [sum(e[2]) for e in eps]},
                   "memory_data/memory{}.pt".format(actor_id))
        mem.load(actor_id)
        assert mem.sequence_counter == int(g["sequence_counter"][i]), f"file {i}"
        tags = []
        for (start, n_rows, n_starts) in mem.memory:
            leaf = torch.tensor([start], dtype=torch.int64, device="cuda")
            obs = torch.empty((65, 1, 4), device="cuda")
            nv.check(mem._dev.lib.r2d2_replay_gather(mem._dev._h, nv.dptr(leaf, torch.int64), 1, nv.dptr(obs), None,
                                                     None, None, None, nv.current_stream()))
            tags.append(int(round(float(obs[0, 0, 0].item()))))
        assert tags == [int(t) for t in g[f"survivors/{i}"]], f"file {i}"
    assert mem._dev.cfg.replay_state_dtype == "float16"
    sys.modules.pop("replay_memory", None)


@pytest.mark.parametrize("max_sequences", [0, 900])
def test_fifo_and_ring_wrap_match_fp32(max_sequences):
    """Files of random episodes through a small ring (it wraps many times) and, in one case, a sequence cap: both modes
    place, evict and count alike, and the windows gathered after the wraps are the rounded originals."""
    cfg = E.PathConfig(obs=5, act=2, hidden=40, batch=8, burn_in=4, learning=6, n_step=2)
    rng = np.random.default_rng(max_sequences)
    cap = 1500
    s32 = E.DeviceReplay(cfg, capacity_rows=cap, max_sequences=max_sequences)
    s16 = E.DeviceReplay(E.PathConfig(**dict(cfg.__dict__, replay_state_dtype="float16")), capacity_rows=cap,
                         max_sequences=max_sequences)
    fed = []
    for f in range(25):
        eps = episodes_with_edges(rng, cfg, int(rng.integers(1, 5)), cfg.rows + 2, cfg.rows + 150)
        r32, r16 = s32.add_episodes(eps), s16.add_episodes(eps)
        assert r32 == r16, f"file {f}"
        a, b = s32.stats(), s16.stats()
        assert a == b, f"file {f}"
        fed += list(zip(r32[0], eps))
    n_live = s16.stats()["n_episodes"]
    live = fed[len(fed) - n_live:]
    leaf = torch.tensor([st + int(rng.integers(0, len(ep[5]))) for st, ep in live], dtype=torch.int64, device="cuda")
    a32, a16 = draw(s32, cfg, "chosen", leaf=leaf), draw(s16, cfg, "chosen", leaf=leaf)
    assert_fp16_draw_is_rounded_fp32_draw(a32, a16)
    for b, (st, ep) in enumerate(live):
        s = int(a16["leaf"][b]) - st
        assert np.array_equal(a16["obs"][:, b], ep[0][s:s + cfg.rows])
        assert_rounded(a16["states"][:, :, b], ep[4][s])
    for l in range(s32.stats()["tree_levels"]):
        assert torch.equal(s32.tree_level(l), s16.tree_level(l)), l
    s32.close()
    s16.close()


# ------------------------------------------------------------------------------------------------ 3. refusal
def _state_of(rp, cfg, u):
    torch.cuda.synchronize()
    return (rp.stats(), [rp.tree_level(l).cpu().numpy().copy() for l in range(rp.stats()["tree_levels"])],
            draw(rp, cfg, "plain", u))


def test_overflowing_file_is_refused_and_changes_nothing():
    cfg = E.PathConfig(obs=5, act=2, hidden=16, batch=8, burn_in=4, learning=6, n_step=2)
    rng = np.random.default_rng(9)
    rp = shard(cfg, "float16", 600, episodes_with_edges(rng, cfg, 6, cfg.rows + 20, cfg.rows + 60))
    u = torch.rand(64, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    for bad in (65520.0, -65520.0, 1e30):
        # a file that would wrap the ring and evict, with one value that fp16 would round to inf in its last episode
        eps = episodes_with_edges(rng, cfg, 3, cfg.rows + 100, cfg.rows + 140)
        eps[-1][4][-1, 3, 1, 5] = bad
        before = _state_of(rp, cfg, u)
        with pytest.raises(nv.NativeError, match="65520"):
            rp.add_episodes(eps)
        with pytest.raises(nv.NativeError, match="65520"):
            rp.add_episode(*eps[-1])
        after = _state_of(rp, cfg, u)
        assert before[0] == after[0]
        for a, b in zip(before[1], after[1]):
            assert np.array_equal(a, b)
        for k in before[2]:
            assert np.array_equal(before[2][k], after[2][k], equal_nan=True), k
    for ok in (65519.99, 65504.0, -65519.99, np.inf, np.nan):
        eps = episodes_with_edges(rng, cfg, 1, cfg.rows + 10, cfg.rows + 12)
        eps[0][4][0, 0, 0, 0] = ok
        starts, _, _ = rp.add_episodes(eps)
        got = draw(rp, cfg, "chosen", leaf=torch.tensor(starts, dtype=torch.int64, device="cuda"))
        assert_rounded(got["states"][:, :, 0], eps[0][4][0])
    rp.close()


# ------------------------------------------------------------------------------------------------ 4. global sampling
def test_global_sampling_w2_fp16():
    """W = 2 in-process ranks: every draw is the restated global draw, the first draw is fp32 storage's, and every
    trained slot holds the rounded rows of its draws."""
    from global_harness import GlobalRun
    kw = dict(obs=7, act=3, hidden=32, batch=16, burn_in=4, learning=6, n_step=2)
    runs, bad = {}, []
    for dtype in ("float32", "float16"):
        run = GlobalRun(E, 2, dict(kw, replay_state_dtype=dtype))

        def on_critic(slot, run=run, dtype=dtype):
            if dtype != "float16":
                return
            shard_of = run.slot_cat("shard", slot).cpu().numpy()
            leaf = run.slot_cat("leaf_idx", slot).cpu().numpy()
            states = run.slot_cat("states", slot).cpu().numpy()
            for k, rp in enumerate(run.shards):
                cols = np.nonzero(shard_of == k)[0]
                ep_i, seq_i = rp.decode(leaf[cols])
                eps = run.episodes[k]
                n_live = rp.stats()["n_episodes"]
                for j, e, s in zip(cols, ep_i, seq_i):
                    want = f16(eps[len(eps) - n_live + e][4][s])
                    if not np.array_equal(states[:, :, j], want):
                        bad.append((k, int(j)))

        run.run(4, prefetch=True, on_critic=on_critic)
        assert run.status() == [0, 0]
        for ref, got in run.draws:
            assert np.array_equal(ref[0], got[0]) and np.array_equal(ref[1], got[1])
        runs[dtype] = [d[1] for d in run.draws]
        run.close()
    assert not bad, bad[:8]
    a, b = runs["float32"][0], runs["float16"][0]
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


# ------------------------------------------------------------------------------------------------ 5. learner
def _gathered_batches(kw, iters, seed):
    """`iters` batches drawn with the same uniforms from an fp32 and an fp16 shard of the same LSTM-like episodes."""
    cfg = E.PathConfig(**kw)
    rng = np.random.default_rng(seed)
    eps = []
    for _ in range(max(8, 2 * cfg.batch // 40)):
        ep = list(episode(rng, cfg, int(rng.integers(cfg.rows + 20, cfg.rows + 120))))
        ep[4] = lstm_like_states(rng, ep[4].shape[0], cfg.hidden)
        eps.append(tuple(ep))
    cap = sum(e[0].shape[0] for e in eps)
    s32, s16 = shard(cfg, "float32", cap, eps), shard(cfg, "float16", cap, eps)
    gen = torch.Generator(device="cuda").manual_seed(seed)
    out = {"float32": [], "float16": []}
    for _ in range(iters):
        u = torch.rand(cfg.batch, device="cuda", generator=gen)
        a32, a16 = draw(s32, cfg, "plain", u), draw(s16, cfg, "plain", u)
        assert_fp16_draw_is_rounded_fp32_draw(a32, a16)
        for dtype, a in (("float32", a32), ("float16", a16)):
            out[dtype].append({"obs": a["obs"], "act": a["act"], "rew": a["rew"], "term": a["term"],
                               **{k: a["states"][i] for i, k in enumerate(("a_state", "ta_state", "c_state", "tc_state"))}})
    s32.close()
    s16.close()
    return out


def _fp16_vs_fp32_run(kw, actor, critic, batches, iters):
    """The same engine on the fp32-storage and the fp16-storage batches: worst relative L2 of q, target and priority per
    iteration and of every net, target and Adam moment at the end."""
    engs = {}
    outs = {d: [] for d in batches}
    for dtype in batches:
        eng = E.LearnerEngine(E.PathConfig(**kw))
        eng.load_state_dicts(actor, critic)
        for it in range(iters):
            eng.set_batch(batches[dtype][it])
            eng.step()
            torch.cuda.synchronize()
            outs[dtype].append({k: getattr(eng, k).cpu().numpy() for k in ("q_value", "target_q_value", "priority")})
        engs[dtype] = eng
    errs = {}
    for it in range(iters):
        for k in outs["float32"][it]:
            errs[f"{k}/{it}"] = rel_l2(outs["float16"][it][k], outs["float32"][it][k])
    for net in ("actor", "critic", "target_actor", "target_critic"):
        for what in ("params", "exp_avg", "exp_avg_sq") if not net.startswith("target") else ("params",):
            a, b = engs["float16"].views(net, what), engs["float32"].views(net, what)
            for k in a:
                errs[f"{what}/{net}/{k}"] = rel_l2(a[k].cpu().numpy(), b[k].cpu().numpy())
    for eng in engs.values():
        eng.close()
    worst = max(errs, key=errs.get)
    return errs[worst], worst, {k: v for k, v in errs.items() if not v < TOL}


@pytest.mark.parametrize("name, iters", [("ref_pend_h128.npz", 12), ("ref_walker_h128.npz", 12), ("cfg2", 6)])
def test_learner_on_fp16_states_against_oracle_and_fp32(name, iters):
    if name == "cfg2":
        kw = dict(obs=17, act=6, hidden=256, batch=256, burn_in=40, learning=80, n_step=5)
        actor, critic, _ = port_case(kw, n_batches=1)
    else:
        kw, actor, critic, _ = golden_case(name)
    batches = _gathered_batches(kw, iters, seed=len(name))
    worst_oracle = check_against_oracle(E, kw, actor, critic, batches["float16"], iters)
    worst, where, bad = _fp16_vs_fp32_run(kw, actor, critic, batches, iters)
    print(f"{name}: fp16 storage vs float64 oracle {worst_oracle:.3e}; vs fp32 storage {worst:.3e} ({where})")
    assert not bad, bad


def _fed_run(make_shard, steps=5, seed=7, kw=None):
    """snapshot() plus launches after `steps` pipelined replay-fed iterations, priorities written back before each draw
    (learner_harness.replay_fed_run with the shard made by make_shard(cfg, cap))."""
    cfg = E.PathConfig(**(kw or REPLAY))
    rng = np.random.default_rng(5)
    eps = []
    for _ in range(24):
        ep = list(episode(rng, cfg, 120))
        ep[4] = lstm_like_states(rng, ep[4].shape[0], cfg.hidden)
        eps.append(tuple(ep))
    rp = make_shard(cfg, 24 * (120 + cfg.n_step))
    rp.add_episodes(eps)
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


def _fp16_shard(cfg, cap):
    return E.DeviceReplay(E.PathConfig(**dict(cfg.__dict__, replay_state_dtype="float16")), capacity_rows=cap)


def test_fp16_pipelined_equals_sequential_and_runs_repeat():
    a = _fed_run(_fp16_shard)
    assert_same_bits(a, _fed_run(_fp16_shard))
    # sequential: draw, step, write back - the pipelined hook's order
    cfg = E.PathConfig(**REPLAY)
    rng = np.random.default_rng(5)
    eps = []
    for _ in range(24):
        ep = list(episode(rng, cfg, 120))
        ep[4] = lstm_like_states(rng, ep[4].shape[0], cfg.hidden)
        eps.append(tuple(ep))
    rp = _fp16_shard(cfg, 24 * (120 + cfg.n_step))
    rp.add_episodes(eps)
    eng = E.LearnerEngine(cfg, seed=7)
    gen = torch.Generator(device="cuda").manual_seed(11)
    for _ in range(5):
        rp.sample_into(eng, generator=gen)
        eng.step()
        rp.update_priorities(eng.leaf_idx, eng.priority)
    b = snapshot(eng)
    b["launches"] = a["launches"]
    assert_same_bits(a, b)
    rp.close()
    eng.close()


# ------------------------------------------------------------------------------------------------ 6. defaults
def _raw_shard(options):
    def make(cfg, cap):
        rp = E.DeviceReplay(cfg, capacity_rows=cap)
        nv.check(rp.lib.r2d2_replay_destroy(rp._h))
        rc = nv.ReplayConfig(cfg.obs, cfg.act, cfg.hidden, cfg.burn_in, cfg.learning, cfg.n_step, int(cap), 0)
        rp._h = c_void_p()
        if options == "create":
            nv.check(rp.lib.r2d2_replay_create(nv.byref(rp._h), nv.byref(rc)))
        elif options is None:
            nv.check(rp.lib.r2d2_replay_create_ex(nv.byref(rp._h), nv.byref(rc), None))
        else:
            nv.check(rp.lib.r2d2_replay_create_ex(nv.byref(rp._h), nv.byref(rc), nv.byref(nv.ReplayOptions(options))))
        return rp
    return make


def test_create_ex_defaults_are_create():
    ref = _fed_run(_raw_shard("create"))
    for opt in (None, nv.STATE_F32):
        assert_same_bits(ref, _fed_run(_raw_shard(opt)))
    assert_same_bits(ref, _fed_run(lambda cfg, cap: E.DeviceReplay(cfg, capacity_rows=cap)))
    rc = nv.ReplayConfig(3, 1, 8, 1, 2, 1, 64, 0)
    h = c_void_p()
    for bad in (2, -1, 16):
        assert nv.lib().r2d2_replay_create_ex(nv.byref(h), nv.byref(rc), nv.byref(nv.ReplayOptions(bad))) != 0


def test_launches_are_equal_in_both_modes():
    a = _fed_run(lambda cfg, cap: E.DeviceReplay(cfg, capacity_rows=cap))
    b = _fed_run(_fp16_shard)
    assert int(a["launches"]) == int(b["launches"])
    cfg = E.PathConfig(**REPLAY)
    rng = np.random.default_rng(1)
    eps = [episode(rng, cfg, 120) for _ in range(4)]
    counts = []
    for dtype in ("float32", "float16"):
        rp = shard(cfg, dtype, 600, eps)
        eng = E.LearnerEngine(cfg)
        for weighted in (False, True):
            eng.importance_weighting = weighted
            n0 = nv.lib().r2d2_launch_count()
            rp.sample_into(eng)
            counts.append((weighted, nv.lib().r2d2_launch_count() - n0))
        rp.close()
        eng.close()
    assert counts[:2] == counts[2:], counts


@pytest.mark.parametrize("H", [512, 36])
def test_device_bytes(H):
    cfg = E.PathConfig(obs=7, act=3, hidden=H, batch=8, burn_in=3, learning=5, n_step=2)
    cap = 3000
    s32, s16 = shard(cfg, "float32", cap), shard(cfg, "float16", cap)
    b32, b16 = s32.device_bytes(), s16.device_bytes()
    assert b32 - b16 == cap * 8 * H * 2
    rng = np.random.default_rng(3)
    eps = episodes_with_edges(rng, cfg, 4, cfg.rows + 100, cfg.rows + 200)
    R = sum(e[0].shape[0] for e in eps)
    for rp in (s32, s16):
        rp.add_episodes(eps)
    assert s32.device_bytes() == b32
    staging = s16.device_bytes() - b16
    assert 4 * R * 8 * H < staging <= 4 * R * 8 * H + 256, staging
    s16.add_episodes(eps[:1])                      # a smaller call reuses the block
    assert s16.device_bytes() - b16 == staging
    s32.close()
    s16.close()

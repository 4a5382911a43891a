"""The replay shard against its host model (oracle/replay_model.py): seeded random sequences of ingests - files of 1 to
6 episodes, many of them wider than the ring so that one call wraps onto its own episodes, and single episodes -
priority write-backs with duplicates and zeros, and snapshot restores at the same and at another capacity, on a
DeviceReplay and on the model side by side.  After every operation:

- stats(), the snapshot counters and the FIFO table are the model's;
- a leaf is nonzero only on a live episode's sequence-start rows, level 0 is the model's p^alpha (bit for bit at
  alpha = 1, 1e-6 relative otherwise) and every upper level is the C sum tree's (oracle/sumtree_oracle.c) over it;
- decode of every row is the model's, the draw on fixed uniforms (0 and 1 - ulp among them) is the C tree's, the
  weighted draw's weights are float64 (min / leaf)^beta, and the gathered windows and start states are the model's rows
  bit for bit (fp16 storage: the rounded states, widened).

Capacities 32 .. 32769 give sum trees of 2 to 5 levels, on both sides of each power of 32."""
import numpy as np
import pytest
import torch

from learner_harness import draw, episode
from oracle.replay_model import ReplayModel
from oracle.sumtree import SumTreeOracle
from r2d2_b200 import engine as E

pytestmark = pytest.mark.gpu

KW = dict(obs=3, act=2, hidden=8, batch=8, burn_in=2, learning=3, n_step=2)   # W = 7 rows; eviction counts 1 more
CAPACITIES = [32, 33, 1023, 1024, 1025, 32768, 32769]                         # levels 2, 3, 3, 3, 4, 4, 5
WRITE_BACKS = [1, 7, 1024, 1025, 5120]
U = np.concatenate([np.float32([0.0, 1.0 - 2.0 ** -24]),
                    np.random.default_rng(0).uniform(size=254).astype(np.float32)])


def shard_episode(rng, cfg, n_rows, full=None):
    """learner_harness.episode of n_rows rows; `full` (default: a coin) gives it the last start too (n_rows - W + 1
    starts instead of n_rows - W), so a one-window episode has 0 or 1 start."""
    ep = episode(rng, cfg, n_rows - cfg.n_step)
    if full is None:
        full = rng.random() < 0.5
    if full:
        ep = ep[:5] + (np.append(ep[5], np.float32(rng.uniform(0.01, 1.0))),)
    return ep


def ring_length(rng, cap, W):
    """One window, the whole ring, or log-uniform in between."""
    r = rng.random()
    if r < 0.15:
        return W
    if r < 0.25:
        return cap
    return int(min(cap, max(W, np.exp(rng.uniform(np.log(W), np.log(cap + 1))))))


def check_against_model(rp, m, cfg, beta=0.6):
    cap = m.capacity
    st = rp.stats()
    want = m.stats()
    assert {k: st[k] for k in want} == want
    info = rp.snapshot_info()
    want = m.info()
    assert {k: info[k] for k in want} == want
    for got, exp, name in zip(rp.episodes(), m.episodes(), ("row_start", "n_rows", "n_starts", "serial")):
        assert np.array_equal(got, exp), name
    levels = [rp.tree_level(l).cpu().numpy() for l in range(st["tree_levels"])]
    lv0 = levels[0]
    stray = np.setdiff1d(np.flatnonzero(lv0), m.live_starts())
    assert stray.size == 0, f"{stray.size} nonzero leaves on rows that start no live sequence: {stray[:10].tolist()}"
    leaves = m.leaves()
    if m.alpha == 1.0:
        assert np.array_equal(lv0[:cap].view(np.uint32), leaves.astype(np.float32).view(np.uint32))
    else:
        assert np.array_equal(lv0[:cap] == 0, leaves == 0)
        pos = leaves > 0
        if pos.any():
            assert np.abs(lv0[:cap][pos] / leaves[pos] - 1.0).max() < 1e-6
    oracle = SumTreeOracle(cap)
    oracle.set_range(0, lv0[:cap])
    assert oracle.levels == len(levels)
    for l in range(1, oracle.levels):
        ol = oracle.level(l)
        assert np.array_equal(levels[l][:ol.size].view(np.uint32), ol.view(np.uint32)), f"level {l}"
    assert st["total_priority"] == oracle.total
    rows = np.arange(cap)
    for got, exp in zip(rp.decode(rows), m.decode(rows)):
        assert np.array_equal(got, exp)
    if not m.fifo:
        return
    u = torch.as_tensor(U).cuda()
    a = draw(rp, cfg, "plain", u)
    assert np.array_equal(a["leaf"], oracle.sample(U))
    for got, exp in zip(rp.decode(a["leaf"]), m.decode(a["leaf"])):
        assert np.array_equal(got, exp)
    if leaves.any():
        assert np.isin(a["leaf"], m.live_starts()).all()
    win = m.window(a["leaf"])
    for k, v in win.items():
        assert np.array_equal(a[k].view(np.uint32), v.view(np.uint32)), k
    w = draw(rp, cfg, "weighted", u, beta=beta)
    for k in win:
        assert np.array_equal(w[k], a[k]), k
    assert np.array_equal(w["leaf"], a["leaf"])
    v = leaves[a["leaf"]]
    want = np.ones(v.size)
    if (v > 0).any():
        want[v > 0] = (v[v > 0].min() / v[v > 0]) ** beta
    assert np.abs(w["w"] - want).max() < 2e-6


def save_and_restore(rp, m, cfg, cap, max_sequences, path):
    rp.save_snapshot(str(path))
    fresh = E.DeviceReplay(cfg, capacity_rows=cap, max_sequences=max_sequences)
    out = fresh.load_snapshot(str(path), restore_rng=False)
    rp.close()
    m, dropped = m.restored(cap)
    assert out["dropped"] == dropped
    return fresh, m


@pytest.mark.parametrize("max_sequences", [0, "cap/3"])
@pytest.mark.parametrize("dtype", ["float32", "float16"])
@pytest.mark.parametrize("alpha", [1.0, 0.6, 0.0])
@pytest.mark.parametrize("cap", CAPACITIES)
def test_random_sequence_against_model(cap, alpha, dtype, max_sequences, tmp_path):
    cfg = E.PathConfig(**KW, priority_exponent=alpha, replay_state_dtype=dtype)
    W = cfg.rows
    ms = cap // 3 if max_sequences else 0
    rng = np.random.default_rng([cap, int(alpha * 10), int(dtype == "float16"), ms])
    rp = E.DeviceReplay(cfg, capacity_rows=cap, max_sequences=ms)
    m = ReplayModel.for_config(cfg, cap, ms)
    ops = ["file"] * 8 + ["wider"] * 4 + ["single"] * 3 + ["write-back"] * 5 + ["restore", "restore-other"]
    rng.shuffle(ops)
    ops = ["wider"] + ops                          # the first call is wider than the ring, on an empty shard
    n_wb = 0
    for i, op in enumerate(ops):
        where = f"op {i} ({op})"
        if op in ("file", "wider"):
            k = int(rng.integers(1, 7) if op == "file" else rng.integers(2, 7))
            if op == "file":
                lens = [ring_length(rng, m.capacity, W) for _ in range(k)]
            else:                                  # k lengths of more than capacity / k rows: the call wraps
                lo = max(W, m.capacity // k + 1)
                lens = [int(n) for n in rng.integers(lo, min(m.capacity, 2 * lo) + 1, k)]
                assert sum(lens) > m.capacity
            eps = [shard_episode(rng, cfg, n) for n in lens]
            assert rp.add_episodes(eps) == m.add_episodes(eps), where
        elif op == "single":
            ep = shard_episode(rng, cfg, ring_length(rng, m.capacity, W))
            rp.add_episode(*ep)
            m.add_episode(*ep)
        elif op == "write-back":
            live = m.live_starts()
            if live.size == 0:
                continue
            n = WRITE_BACKS[n_wb % len(WRITE_BACKS)]
            n_wb += 1
            leaf = rng.choice(live, n)                                  # with replacement: duplicates
            if n > 1:
                leaf[-(n // 4 + 1):] = leaf[:n // 4 + 1]
            prio = rng.uniform(0.01, 2.0, n).astype(np.float32)
            prio[rng.random(n) < 0.1] = 0
            rp.update_priorities(torch.as_tensor(leaf).cuda(), torch.as_tensor(prio).cuda())
            m.update_priorities(leaf, prio)
        else:
            new_cap = m.capacity
            if op == "restore-other":              # smaller (the oldest may not fit) or larger
                new_cap = max(W, 2 * m.capacity // 3) if rng.random() < 0.5 else m.capacity + m.capacity // 3 + 1
            rp, m = save_and_restore(rp, m, cfg, new_cap, ms, tmp_path / f"shard{i}.snap")
        try:
            check_against_model(rp, m, cfg, beta=(0.6, 1.0)[i % 2])
        except AssertionError as e:
            raise AssertionError(f"{where}: {e}") from e
    rp.close()


@pytest.mark.parametrize("dtype", ["float32", "float16"])
def test_call_that_wraps_onto_its_own_episode(dtype, tmp_path):
    """400 + 400 + 300 rows in one call to an empty ring of 1000 (W = 6): the third episode wraps to row 0 and evicts
    the first, which the same call placed.  The first episode's start rows past the third (300 .. 394) must hold no
    priority: nothing could decode them, their windows are stale, and a snapshot - which keeps live episodes only -
    would change the draw law."""
    cfg = E.PathConfig(**dict(KW, n_step=1, replay_state_dtype=dtype))
    rng = np.random.default_rng(400)
    rp = E.DeviceReplay(cfg, capacity_rows=1000)
    m = ReplayModel.for_config(cfg, 1000)
    eps = [shard_episode(rng, cfg, n, full=True) for n in (400, 400, 300)]
    assert rp.add_episodes(eps) == m.add_episodes(eps) == ([0, 400, 0], 1, 395 + 395 + 295 - 395)
    check_against_model(rp, m, cfg)
    u = torch.as_tensor(U).cuda()
    before = draw(rp, cfg, "plain", u)
    rp, m = save_and_restore(rp, m, cfg, 1000, 0, tmp_path / "shard.snap")
    check_against_model(rp, m, cfg)
    after = draw(rp, cfg, "plain", u)
    for k in before:
        assert np.array_equal(before[k], after[k]), k
    rp.close()

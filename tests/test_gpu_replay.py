"""GPU replay shard: sum-tree indices bit-exact against the C restatement (oracle/sumtree_oracle.c),
gather correctness, duplicate handling, eviction, and the sampling distribution against the reference's
two-level sampler (fixture tests/golden/ref_sampler_hist.npz)."""
import os

import numpy as np
import pytest
import torch

from conftest import load_golden
from learner_harness import episode
from oracle.sumtree import SumTreeOracle

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng_mod():
    from r2d2_b200 import engine
    return engine


def fill(rp, oracle, rng, cfg, lens):
    eps, row = [], 0
    for E in lens:
        ep = episode(rng, cfg, E, zero_pad=True)
        rp.add_episode(*ep)
        n_rows = ep[0].shape[0]
        oracle.set_range(row, ep[5])
        oracle.set_range(row + len(ep[5]), None, n_rows - len(ep[5]))
        eps.append((row, ep))
        row += n_rows
    return eps


def test_tree_bit_exact_and_gather(eng_mod):
    cfg = eng_mod.PathConfig(obs=5, act=2, hidden=32, batch=64, burn_in=6, learning=10, n_step=3)
    rng = np.random.default_rng(0)
    cap = 40000
    rp = eng_mod.DeviceReplay(cfg, capacity_rows=cap)
    oracle = SumTreeOracle(cap)
    lens = list(rng.integers(20, 400, size=120))
    eps = fill(rp, oracle, rng, cfg, lens)
    st = rp.stats()
    assert st["n_episodes"] == len(lens) and st["tree_levels"] == oracle.levels
    for l in range(oracle.levels):
        assert np.array_equal(rp.tree_level(l).cpu().numpy()[:len(oracle.level(l))], oracle.level(l)), f"level {l}"
    # --- sampling: identical indices for identical uniforms (incl. the edges of [0,1))
    u = np.concatenate([rng.uniform(size=20000).astype(np.float32), np.float32([0.0, np.nextafter(np.float32(1), np.float32(0))])])
    leaf = rp.sample_indices(torch.as_tensor(u).cuda()).cpu().numpy()
    assert np.array_equal(leaf, oracle.sample(u))
    leaves0 = oracle.level(0)
    assert (leaves0[leaf] > 0).all()
    # --- gather: time-major window + stored recurrent state of the start row
    eng = eng_mod.LearnerEngine(cfg)
    rp.sample_into(eng, u=torch.as_tensor(u[:cfg.batch]).cuda())
    torch.cuda.synchronize()
    li = eng.leaf_idx.cpu().numpy()
    assert np.array_equal(li, oracle.sample(u[:cfg.batch]))
    ep_i, seq_i = rp.decode(li)
    obs, act, rew, term, states = (t.cpu().numpy() for t in (eng.obs, eng.act, eng.rew, eng.term, eng.states))
    for b in range(cfg.batch):
        row0, ep = eps[ep_i[b]]
        s = seq_i[b]
        assert row0 + s == li[b]
        assert np.array_equal(obs[:, b], ep[0][s:s + cfg.rows])
        assert np.array_equal(act[:, b], ep[1][s:s + cfg.rows])
        assert np.array_equal(rew[:, b], ep[2][s:s + cfg.rows])
        assert np.array_equal(term[:, b], ep[3][s:s + cfg.rows])
        assert np.array_equal(states[:, :, b], ep[4][s])
    # --- priority write-back with duplicates: last writer wins, ancestors recomputed
    upd_leaf = np.concatenate([li[:40], li[:8]])
    upd_p = rng.uniform(0.5, 3.0, upd_leaf.size).astype(np.float32)
    rp.update_priorities(torch.as_tensor(upd_leaf).cuda(), torch.as_tensor(upd_p).cuda())
    oracle.update_batch(upd_leaf, upd_p)
    for l in range(oracle.levels):
        assert np.array_equal(rp.tree_level(l).cpu().numpy()[:len(oracle.level(l))], oracle.level(l)), f"level {l}"
    u2 = rng.uniform(size=5000).astype(np.float32)
    assert np.array_equal(rp.sample_indices(torch.as_tensor(u2).cuda()).cpu().numpy(), oracle.sample(u2))


def test_distribution_matches_reference_sampler(eng_mod):
    """P(start) proportional to priority: same law as the reference's two-level draw (chi-square vs the
    priorities, with the reference's own histogram from the fixture passing the same test)."""
    g = load_golden("ref_sampler_hist.npz")
    pri, offs = g["priorities"].astype(np.float32), g["episode_offsets"]
    cfg = eng_mod.PathConfig(obs=3, act=1, hidden=4, batch=32)  # burn_in 20, learning 40, n 5 like the fixture
    rp = eng_mod.DeviceReplay(cfg, capacity_rows=4096)
    rows, starts = [], []
    row = 0
    for e in range(len(offs) - 1):
        p = pri[offs[e]:offs[e + 1]]
        E = len(p) + 60
        n_rows = E + 5
        rp.add_episode(np.zeros((n_rows, 3), np.float32), np.zeros((n_rows, 1), np.float32), np.zeros(n_rows, np.float32),
                       np.zeros(n_rows, np.float32), np.zeros((E, 4, 2, 4), np.float32), p)
        starts.append(row + np.arange(len(p)))
        row += n_rows
    starts = np.concatenate(starts)
    n = 400000
    u = torch.rand(n, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    leaf = rp.sample_indices(u).cpu().numpy()
    cnt = np.bincount(leaf, minlength=row)
    assert cnt.sum() == cnt[starts].sum()          # only valid sequence starts are ever drawn
    exp = pri.astype(np.float64) / pri.astype(np.float64).sum() * n
    chi2 = ((cnt[starts] - exp) ** 2 / exp).sum() / len(pri)
    assert 0.7 < chi2 < 1.3, chi2
    exp_ref = pri.astype(np.float64) / pri.astype(np.float64).sum() * int(g["n_draws"])
    chi2_ref = ((g["counts"] - exp_ref) ** 2 / exp_ref).sum() / len(pri)
    assert 0.7 < chi2_ref < 1.3, chi2_ref


def test_fifo_eviction(eng_mod):
    cfg = eng_mod.PathConfig(obs=4, act=2, hidden=8, batch=8, burn_in=4, learning=6, n_step=2)
    rng = np.random.default_rng(5)
    rp = eng_mod.DeviceReplay(cfg, capacity_rows=1000)
    oracle = SumTreeOracle(1000)
    live, head = [], 0
    for i in range(30):
        E = int(rng.integers(30, 120))
        ep = episode(rng, cfg, E, zero_pad=True)
        n_rows = E + cfg.n_step
        if head + n_rows > 1000:
            head = 0
        while live and live[0][0] < head + n_rows and head < live[0][0] + live[0][1]:
            r0, nr, ns = live.pop(0)
            oracle.set_range(r0, None, ns)
        rp.add_episode(*ep)
        oracle.set_range(head, ep[5])
        oracle.set_range(head + len(ep[5]), None, n_rows - len(ep[5]))
        live.append((head, n_rows, len(ep[5])))
        head += n_rows
        assert rp.stats()["n_episodes"] == len(live)
    for l in range(oracle.levels):
        assert np.array_equal(rp.tree_level(l).cpu().numpy()[:len(oracle.level(l))], oracle.level(l))
    u = rng.uniform(size=4000).astype(np.float32)
    leaf = rp.sample_indices(torch.as_tensor(u).cuda()).cpu().numpy()
    assert np.array_equal(leaf, oracle.sample(u))
    ep_i, _ = rp.decode(leaf)
    assert (ep_i >= 0).all()


def test_large_tree_bit_exact(eng_mod):
    """cfg-4 scale shard: 250k sequence starts (1,000 episodes x 250), indices identical to the C tree."""
    cfg = eng_mod.PathConfig(obs=2, act=1, hidden=4, batch=512)
    n_ep, E = 1000, 310
    cap = n_ep * (E + 5)
    rp = eng_mod.DeviceReplay(cfg, capacity_rows=cap)
    oracle = SumTreeOracle(cap)
    rng = np.random.default_rng(9)
    zo = np.zeros((E + 5, 2), np.float32)
    za = np.zeros((E + 5, 1), np.float32)
    zr = np.zeros(E + 5, np.float32)
    zs = np.zeros((E, 4, 2, 4), np.float32)
    row = 0
    for _ in range(n_ep):
        p = rng.uniform(0.01, 1.0, E - 60).astype(np.float32)
        rp.add_episode(zo, za, zr, zr, zs, p)
        oracle.set_range(row, p)
        row += E + 5
    u = rng.uniform(size=100000).astype(np.float32)
    leaf = rp.sample_indices(torch.as_tensor(u).cuda()).cpu().numpy()
    assert np.array_equal(leaf, oracle.sample(u))
    for _ in range(3):
        upd = leaf[rng.integers(0, leaf.size, 512)]
        pr = rng.uniform(0.01, 2.0, 512).astype(np.float32)
        rp.update_priorities(torch.as_tensor(upd).cuda(), torch.as_tensor(pr).cuda())
        oracle.update_batch(upd, pr)
    u = rng.uniform(size=100000).astype(np.float32)
    assert np.array_equal(rp.sample_indices(torch.as_tensor(u).cuda()).cpu().numpy(), oracle.sample(u))
    assert abs(rp.stats()["total_priority"] - oracle.total) == 0.0


def test_ingest_matches_reference_load_sequence(tmp_path, monkeypatch):
    """Next-row N1: the same sequence of actor files through the drop-in LearnerReplayMemory.load and through the
    UNMODIFIED reference (fixture tests/golden/ref_ingest.npz, oracle/make_golden.py gen_ingest): sequence_counter -
    incl. the asymmetric eviction arithmetic of replay_memory.py:147 vs :149 - and the surviving episodes after every
    file.  The file is consumed (claimed by rename, removed) instead of rewritten empty."""
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
                                        obs_size=4, n_actions=2, hidden=8, capacity_rows=4096)
    for i, (actor_id, eps) in enumerate(ingest_file_sequence()):
        torch.save({"replay_memory": deque([e[0] for e in eps]), "recurrent_state": deque([e[1] for e in eps]),
                    "priority": deque([e[2] for e in eps]), "total_priority": [sum(e[2]) for e in eps]},
                   "memory_data/memory{}.pt".format(actor_id))
        mem.load(actor_id)
        assert not os.path.exists("memory_data/memory{}.pt".format(actor_id))
        assert mem.sequence_counter == int(g["sequence_counter"][i]), f"file {i}"
        # surviving episodes: the tag stored in obs[0] of each episode's first row, read back from HBM
        tags = []
        for (start, n_rows, n_starts) in mem.memory:
            leaf = torch.tensor([start], dtype=torch.int64, device="cuda")
            obs = torch.empty((65, 1, 4), device="cuda")
            from r2d2_b200 import native as nv
            # gather the window that starts at the episode's first row (explicit leaf, no draw)
            nv.check(mem._dev.lib.r2d2_replay_gather(mem._dev._h, nv.dptr(leaf, torch.int64), 1, nv.dptr(obs), None, None,
                                                     None, None, nv.current_stream()))
            tags.append(int(round(float(obs[0, 0, 0].item()))))
        assert tags == [int(t) for t in g[f"survivors/{i}"]], f"file {i}"
    sys.modules.pop("replay_memory", None)


def test_ring_wrap_evicts_until_no_overlap(eng_mod):
    engine = eng_mod
    """ADVICE r1: oldest episode at the tail of the ring, a younger one at the head that the wrapped episode overwrites:
    both must be evicted (FIFO), not an error."""
    cfg = engine.PathConfig(obs=3, act=1, hidden=8, batch=2, burn_in=2, learning=3, n_step=1)   # window = 6 rows
    rp = engine.DeviceReplay(cfg, capacity_rows=100)
    rng = np.random.default_rng(0)

    def ep(n):
        return (rng.standard_normal((n, 3)).astype(np.float32), rng.uniform(-1, 1, (n, 1)).astype(np.float32),
                rng.standard_normal(n).astype(np.float32), np.zeros(n, np.float32),
                np.zeros((n - 1, 4, 2, 8), np.float32), rng.uniform(0.1, 1, n - 5).astype(np.float32))
    rp.add_episodes([ep(60)])            # A @ [0, 60)
    rp.add_episodes([ep(40)])            # F @ [60, 100)
    rp.add_episodes([ep(50)])            # G wraps to [0, 50): evicts A
    st = rp.stats()
    assert st["n_episodes"] == 2
    starts, n_evicted, _ = rp.add_episodes([ep(60)])   # does not fit behind G (50 + 60 > 100): wraps to [0, 60) -> F then G go
    assert starts == [0] and n_evicted == 2
    assert rp.stats()["n_episodes"] == 1
    leaves = rp.tree_level(0).cpu().numpy()
    assert (leaves[60:] == 0).all() and abs(float(rp.tree_level(rp.stats()["tree_levels"] - 1)[0]) - leaves[:55].sum()) < 1e-4

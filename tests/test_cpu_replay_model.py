"""The host model of a replay shard (oracle/replay_model.py) on its own: the reference's file sequence
(tests/golden/ref_ingest.npz, made by the unmodified LearnerReplayMemory.load) pins its counter arithmetic and FIFO
order, and hand-worked rings pin placement, wrap, eviction, the sequence cap, decode and snapshot restore."""
import numpy as np
import pytest

from conftest import load_golden
from oracle.make_golden import ingest_file_sequence
from oracle.replay_model import ReplayModel

W6 = dict(obs=3, act=2, hidden=4, burn_in=2, learning=3, n_step=1)   # window W = 6 rows: n - 5 starts at most


def ep(n, tag=0.0, n_starts=None, hidden=4):
    """An episode of n rows whose obs hold tag + row / 1000 and whose starts have priority 1 + row / 1000."""
    k = n - 5 if n_starts is None else n_starts
    obs = (tag + np.arange(n, dtype=np.float32) / 1000)[:, None].repeat(3, 1)
    return (obs, np.zeros((n, 2), np.float32), np.arange(n, dtype=np.float32), np.zeros(n, np.float32),
            np.full((n - 1, 4, 2, hidden), tag, np.float32), 1 + np.arange(k, dtype=np.float32) / 1000)


def model(cap, max_sequences=0, **kw):
    return ReplayModel(cap, **dict(W6, **kw), max_sequences=max_sequences)


def table(m):
    return [tuple(int(x) for x in e) for e in m.fifo]


def nonzero_leaves(m):
    return np.flatnonzero(m.leaves())


# ------------------------------------------------------------------------------------------------ 1. the reference
def test_reference_file_sequence():
    """Every file of ingest_file_sequence() through the model with a ring that never wraps: the reference's sequence
    counter and surviving episodes (the tag in obs[0] of each first row) after every file."""
    g = load_golden("ref_ingest.npz")
    files = ingest_file_sequence()
    rows = sum(len(e[0]) for _, eps in files for e in eps)
    m = ReplayModel(rows, obs=4, act=2, hidden=8, burn_in=20, learning=40, n_step=5,
                    max_sequences=int(g["memory_sequence_size"]))
    for i, (_, eps) in enumerate(files):
        batch = []
        for rows_, st, pr, _tag in eps:
            batch.append((np.stack([r[0] for r in rows_]), np.stack([r[1] for r in rows_]),
                          np.float32([r[2][0] for r in rows_]), np.float32([r[3][0] for r in rows_]),
                          np.asarray(st, np.float32), np.float32(pr)))
        _, _, counter = m.add_episodes(batch)
        assert counter == m.sequence_counter == int(g["sequence_counter"][i]), f"file {i}"
        tags = [int(round(float(m.obs[s, 0]))) for s, _, _, _ in m.fifo]
        assert tags == [int(t) for t in g[f"survivors/{i}"]], f"file {i}"
    assert m.evicted_total > 0                                   # the cap evicted
    s0 = m.fifo[0][0]
    assert m.head == rows and m.head - s0 == m.rows_used         # no wrap: the survivors are the ring's last rows


# ------------------------------------------------------------------------------------------------ 2. the ring
def test_plain_wrap():
    m = model(100)
    assert m.add_episodes([ep(60, 1)]) == ([0], 0, 55)
    assert m.add_episodes([ep(30, 2)]) == ([60], 0, 80)
    # 90 + 20 > 100: row 0, which the first episode holds; it goes, with the reference's count (60 - 5)
    assert m.add_episodes([ep(20, 3)]) == ([0], 1, 80 + 15 - 55)
    assert table(m) == [(60, 30, 25, 1), (0, 20, 15, 2)]
    assert (m.head, m.rows_used, m.evicted_total, m.next_serial) == (20, 50, 1, 3)
    assert np.array_equal(nonzero_leaves(m), np.r_[0:15, 60:85])
    assert np.array_equal(m.live_starts(), np.r_[0:15, 60:85])
    ep_i, seq = m.decode([0, 19, 20, 59, 60, 89, 90, 99])
    assert ep_i.tolist() == [1, 1, -1, -1, 0, 0, -1, -1] and seq.tolist() == [0, 19, -1, -1, 0, 29, -1, -1]
    # rows of the evicted episode stay where nothing overwrote them; a window is T consecutive rows
    assert m.obs[30, 0] == np.float32(1 + 30 / 1000)
    w = m.window([60, 2])
    assert w["obs"].shape == (6, 2, 3) and w["states"].shape == (4, 2, 2, 4)
    assert np.array_equal(w["obs"][:, 0, 0], np.float32(2 + np.arange(6) / 1000))
    assert np.array_equal(w["rew"][:, 1], np.float32(np.arange(2, 8)))
    assert (w["states"][:, :, 0] == 2).all() and (w["states"][:, :, 1] == 3).all()


def test_wrap_evicts_old_tail_and_young_head():
    """After a wrap the oldest episode sits at the tail and a younger one at the head: a wrapped episode that overlaps
    the younger one evicts both, front first."""
    m = model(100)
    m.add_episodes([ep(60, 1)])                                   # A [0, 60)
    m.add_episodes([ep(40, 2)])                                   # F [60, 100)
    assert m.add_episodes([ep(50, 3)])[:2] == ([0], 1)            # G wraps to [0, 50), A goes
    assert m.add_episodes([ep(60, 4)])[:2] == ([0], 2)            # 50 + 60 > 100: wraps again, F then G go
    assert table(m) == [(0, 60, 55, 3)]
    assert m.sequence_counter == (55 + 35 + 45 + 55) - (55 + 35 + 45)
    assert np.array_equal(nonzero_leaves(m), np.r_[0:55])


def test_one_call_wraps_onto_its_own_episodes():
    """400 + 400 + 300 rows in one call to a ring of 1000: the third wraps to row 0 and evicts the first, which the same
    call placed.  Its start rows past the third episode (300 .. 394) belong to nobody and must hold no priority."""
    m = model(1000)
    got = m.add_episodes([ep(400, 1, 395), ep(400, 2, 395), ep(300, 3, 295)])
    assert got == ([0, 400, 0], 1, 395 + 395 + 295 - 395)
    assert table(m) == [(400, 400, 395, 1), (0, 300, 295, 2)]
    assert (m.head, m.rows_used) == (300, 700)
    assert np.array_equal(nonzero_leaves(m), np.r_[0:295, 400:795])
    assert not m.raw[300:400].any()
    assert (m.decode(np.arange(300, 400))[0] == -1).all()


def test_one_call_wraps_twice():
    m = model(100)
    starts, n_ev, _ = m.add_episodes([ep(60, 1), ep(70, 2), ep(80, 3)])
    assert (starts, n_ev) == ([0, 0, 0], 2)
    assert table(m) == [(0, 80, 75, 2)]
    assert np.array_equal(m.obs[:80, 0], np.float32(3 + np.arange(80) / 1000))


@pytest.mark.parametrize("route", ["file", "single"])
def test_sequence_cap_can_empty_the_shard(route):
    """The cap applies after the call and pops while the counter exceeds it, whatever is left - also the call's own
    and only episode.  Both ingest routes follow the rule."""
    m = model(100, max_sequences=10)
    add = (lambda e: m.add_episodes([e])) if route == "file" else (lambda e: m.add_episode(*e))
    assert add(ep(30, 1)) == ([0], 1, 0)                          # 25 > 10: evicted by its own call
    assert not m.fifo and m.rows_used == 0 and not m.raw.any()
    assert m.head == 30                                           # eviction does not move the head
    assert add(ep(12, 2)) == ([30], 0, 7)
    assert add(ep(9, 3)) == ([42], 1, 7 + 4 - 7)                  # 11 > 10: the oldest goes, 9 - 5 = 4 stays
    assert table(m) == [(42, 9, 4, 2)]


def test_write_back_last_writer_wins_and_alpha():
    m = model(100, alpha=0.5)
    m.add_episodes([ep(20, 1)])
    m.update_priorities([3, 4, 3, 5], np.float32([9.0, 0.0, 4.0, 0.25]))
    lv = m.leaves()
    assert lv[3] == 2.0 and lv[4] == 0.0 and lv[5] == 0.5
    assert np.array_equal(np.flatnonzero(lv), np.r_[0:4, 5:15])
    assert model(100, alpha=0.0).leaves().sum() == 0
    z = model(100, alpha=0.0)
    z.add_episodes([ep(20, 1)])
    z.update_priorities([7], np.float32([0.0]))
    assert np.array_equal(z.leaves()[:15], np.float64([1] * 7 + [0] + [1] * 7))


def test_fp16_states_are_rounded_once():
    m = model(100, state_f16=True)
    e = list(ep(20, 1))
    e[4] = np.full((19, 4, 2, 4), 1 + 2.0 ** -12, np.float32)      # not an fp16 value: rounds to 1
    m.add_episodes([tuple(e)])
    assert (m.states[:19] == 1).all() and (m.states[19] == 0).all()


# ------------------------------------------------------------------------------------------------ 3. restore
def test_restore_same_capacity_is_the_same_shard():
    m = model(100)
    for n, t in ((60, 1), (30, 2), (20, 3)):
        m.add_episodes([ep(n, t)])
    m.update_priorities([61, 61], np.float32([5.0, 7.0]))
    r, dropped = m.restored(100)
    assert dropped == 0
    assert table(r) == table(m) and r.info() == m.info()
    live = np.zeros(100, bool)
    for s, n, _, _ in m.fifo:
        live[s:s + n] = True
    for k in ("obs", "act", "rew", "term", "states", "raw"):
        a, b = getattr(r, k), getattr(m, k)
        assert np.array_equal(a[live], b[live]) and not a[~live].any(), k
    assert r.raw[61] == 7.0


def test_restore_other_capacity_packs_and_drops_the_oldest():
    m = model(100)
    for n, t in ((60, 1), (30, 2), (20, 3)):
        m.add_episodes([ep(n, t)])                                 # FIFO: (60, 30), (0, 20)
    big, dropped = m.restored(200)
    assert dropped == 0 and table(big) == [(0, 30, 25, 1), (30, 20, 15, 2)]
    assert (big.head, big.rows_used, big.sequence_counter, big.evicted_total) == (50, 50, m.sequence_counter, 1)
    assert np.array_equal(big.obs[:30], m.obs[60:90]) and np.array_equal(big.obs[30:50], m.obs[:20])
    assert np.array_equal(big.raw[:50], np.r_[m.raw[60:90], m.raw[:20]])
    small, dropped = m.restored(45)
    assert dropped == 1 and table(small) == [(0, 20, 15, 2)]
    assert (small.head, small.rows_used, small.evicted_total) == (20, 20, 2)
    assert small.sequence_counter == m.sequence_counter - (30 - 5)
    none, dropped = m.restored(10)
    assert dropped == 2 and not none.fifo and none.head == 0 and none.rows_used == 0

"""Replay snapshots, host side: the file header and episode table round-trip; a truncated file, a bad magic or version,
other sizes, another alpha and another world size are refused before the shard is touched; R2D2_REPLAY_SNAPSHOT_INTERVAL
takes 0 and multiples of 50 only; the training loop calls the snapshot hook only after the ingest of its steps, never
with a batch in flight, and without the hook makes today's calls; the restore kernels keep everything in registers."""
import os

import numpy as np
import pytest

from learner_harness import fake_engine_learner
from sass_report import functions, library_sass, ops, ptxas_report


def _header(**kw):
    from r2d2_b200 import replay_snapshot as rs
    base = dict(obs_size=5, n_actions=2, hidden=8, burn_in=3, learning=4, n_step=2, state_storage=1,
                priority_exponent=0.9, capacity_rows=500, max_sequences=10_000, n_episodes=3, head=321,
                sequence_counter=77, next_serial=12, evicted_total=9, rows_used=90, world=2, rank=1, learner_step=150,
                chunk_rows=7, rng_state=bytes(range(16)) * 3)
    base.update(kw)
    return rs.Header(**base)


TABLE = (np.array([100, 140, 250], np.int64), np.array([40, 20, 30], np.int32), np.array([30, 12, 22], np.int32),
         np.array([9, 10, 11], np.int64))


def _write(path, h, table=TABLE, rows_bytes=None):
    from r2d2_b200 import replay_snapshot as rs
    with open(path, "wb") as f:
        f.write(h.to_bytes())
        f.write(rs.pack_episodes(*table))
        f.write(b"\0" * (h.rows_used * h.row_bytes() if rows_bytes is None else rows_bytes))


def test_header_and_episode_table_round_trip(tmp_path):
    from r2d2_b200 import replay_snapshot as rs
    h = _header()
    p = tmp_path / "s"
    _write(p, h)
    with open(p, "rb") as f:
        back = rs.Header.read(f)
        table = rs.read_episodes(f, back)
    assert back.priority_exponent == float(np.float32(0.9))   # held as float32, as the shard holds alpha
    back.priority_exponent = h.priority_exponent
    assert back == h
    for k, col in zip(("row_start", "n_rows", "n_starts", "serial"), TABLE):
        assert table[k].tolist() == col.tolist()
    # rows: 4 (O + A + rew + term + leaf) floats and 8 H states of 2 (fp16) or 4 bytes
    assert h.row_bytes() == 4 * (5 + 2 + 3) + 2 * 8 * 8
    assert _header(state_storage=0).row_bytes() == 4 * (5 + 2 + 3) + 4 * 8 * 8
    assert os.path.getsize(p) == h.file_bytes()


class _Untouchable:
    """A shard whose native side must not be reached: any use of its library fails the test."""

    def __init__(self, **cfg):
        from r2d2_b200 import engine
        self.cfg = engine.PathConfig(**dict(dict(obs=5, act=2, hidden=8, burn_in=3, learning=4, n_step=2,
                                                 priority_exponent=0.9), **cfg))

    @property
    def lib(self):
        raise AssertionError("the shard was touched before the snapshot was refused")

    _h = property(lib.fget)


def _refused(path, match, world=None, **cfg):
    from r2d2_b200 import replay_snapshot as rs
    with pytest.raises(ValueError, match=match):
        rs.load(_Untouchable(**cfg), str(path), world=world)


def test_a_whole_file_passes_the_checks(tmp_path):
    from r2d2_b200 import replay_snapshot as rs
    p = tmp_path / "s"
    _write(p, _header())
    h, table = rs.read_checked(str(p), (5, 2, 8, 3, 4, 2), 0.9, world=2)
    assert h.n_episodes == len(table) == 3


def test_truncated_files_are_refused_before_the_shard_is_touched(tmp_path):
    h = _header()
    full = h.rows_used * h.row_bytes()
    for i, rows in enumerate((full - 1, 0, full // 2, full + 4)):     # short rows, no rows, a longer file
        p = tmp_path / f"rows{i}"
        _write(p, h, rows_bytes=rows)
        _refused(p, "truncated or damaged")
    p = tmp_path / "table"
    with open(p, "wb") as f:
        f.write(h.to_bytes())
        f.write(b"\0" * 10)
    _refused(p, "truncated")
    p = tmp_path / "header"
    with open(p, "wb") as f:
        f.write(h.to_bytes()[:30])
    _refused(p, "truncated header")


def test_bad_magic_and_version_are_refused(tmp_path):
    from r2d2_b200 import replay_snapshot as rs
    raw = bytearray(_header().to_bytes())
    p = tmp_path / "magic"
    with open(p, "wb") as f:
        f.write(b"NOTASNAP" + raw[8:])
    _refused(p, "not a replay snapshot")
    p = tmp_path / "version"
    with open(p, "wb") as f:
        f.write(raw[:8] + (rs.VERSION + 1).to_bytes(4, "little") + raw[12:])
    _refused(p, "format version")


@pytest.mark.parametrize("field, value", [("obs", 6), ("act", 3), ("hidden", 16), ("burn_in", 2), ("learning", 5),
                                          ("n_step", 3)])
def test_other_sizes_are_refused(tmp_path, field, value):
    p = tmp_path / "s"
    _write(p, _header())
    _refused(p, "obs / act / hidden", **{field: value})


def test_another_alpha_is_refused(tmp_path):
    p = tmp_path / "s"
    _write(p, _header())
    for alpha in (1.0, 0.6, 0.0):
        _refused(p, "priority exponent", priority_exponent=alpha)


def test_another_world_size_is_refused_naming_both(tmp_path):
    p = tmp_path / "s"
    _write(p, _header(world=2))
    _refused(p, "world size 2, this run has world size 4", world=4)


def test_snapshot_interval_variable():
    from learner import snapshot_interval_from_environ as parse
    assert parse({}) == 0
    for ok in (0, 50, 100, 500, 5000):
        assert parse({"R2D2_REPLAY_SNAPSHOT_INTERVAL": str(ok)}) == ok
    for bad in ("25", "75", "1", "-50", "x", "50.0", "", "1e2"):
        with pytest.raises(ValueError, match="R2D2_REPLAY_SNAPSHOT_INTERVAL"):
            parse({"R2D2_REPLAY_SNAPSHOT_INTERVAL": bad})


def test_learner_reads_the_snapshot_interval(monkeypatch, tmp_path):
    assert fake_engine_learner(monkeypatch, tmp_path).replay_snapshot_interval == 0
    assert fake_engine_learner(monkeypatch, tmp_path, R2D2_REPLAY_SNAPSHOT_INTERVAL="100").replay_snapshot_interval == 100
    with pytest.raises(ValueError, match="R2D2_REPLAY_SNAPSHOT_INTERVAL"):
        fake_engine_learner(monkeypatch, tmp_path, R2D2_REPLAY_SNAPSHOT_INTERVAL="30")


def test_latest_complete_snapshot(tmp_path):
    from learner import latest_complete_snapshot, snapshot_steps
    root = tmp_path / "replay_snapshot"
    assert latest_complete_snapshot(str(root)) is None
    for step, complete in ((50, True), (100, True), (150, False), (1000, False)):
        d = root / f"step{step}"
        d.mkdir(parents=True)
        if complete:
            (d / "COMPLETE").write_text(str(step))
    (root / "stepx").mkdir()
    (root / "step7.tmp").mkdir()
    assert [s for s, _ in snapshot_steps(str(root))] == [50, 100, 150, 1000]
    assert latest_complete_snapshot(str(root)) == (100, str(root / "step100"))


# ---------------------------------------------------------------------------------------------- training loop
class _Engine:
    """Mimics LearnerEngine.step: the prefetch hook runs once per step, after the priorities of the batch exist."""

    def __init__(self, log):
        self.log, self.batch, self.leaf_idx, self.priority = log, None, None, None

    def step(self, prefetch=None):
        trained = self.batch
        assert trained is not None
        self.log.append(("step", trained, prefetch is not None))
        self.leaf_idx, self.priority = trained, trained
        self.batch = None
        if prefetch is not None:
            from types import SimpleNamespace
            prefetch(self, SimpleNamespace(leaf_idx=trained, priority=trained))


class _Replay:
    def __init__(self, log):
        self.log, self.draws = log, 0

    def sample_into(self, eng):
        self.draws += 1
        eng.batch = self.draws
        self.log.append(("draw", self.draws))

    def update_priorities(self, leaf_idx, priority):
        self.log.append(("writeback", leaf_idx))


def _run(max_steps, ingest_every, save_every, snapshot_every=None):
    from r2d2_b200.run_loop import run_learner_loop
    log = []
    eng, rp = _Engine(log), _Replay(log)
    kw = {}
    if snapshot_every is not None:
        def snapshot():
            # nothing in flight: the engine holds no prefetched batch and every trained batch is written back
            assert eng.batch is None
            draws = [e[1] for e in log if e[0] == "draw"]
            backs = [e[1] for e in log if e[0] == "writeback"]
            assert backs == draws
            log.append(("snapshot",))
        kw = dict(snapshot=snapshot, snapshot_every=snapshot_every)
    run_learner_loop(eng, rp, max_steps=max_steps, ingest_every=ingest_every, save_every=save_every,
                     ingest=lambda: log.append(("ingest",)), save=lambda: log.append(("save",)),
                     log=lambda s: log.append(("log", s)), log_every=5, **kw)
    return log


@pytest.mark.parametrize("max_steps, ingest_every, save_every, snapshot_every",
                         [(23, 5, 4, 10), (12, 1, 3, 4), (150, 50, 50, 50), (31, 3, 7, 3), (9, 4, 4, 8)])
def test_snapshot_hook_runs_after_the_ingest_of_its_steps(max_steps, ingest_every, save_every, snapshot_every):
    log = _run(max_steps, ingest_every, save_every, snapshot_every)
    at = [i for i, e in enumerate(log) if e == ("snapshot",)]
    assert len(at) == max_steps // snapshot_every
    for i in at:
        assert log[i - 1] == ("ingest",)
        steps = [e for e in log[:i] if e[0] == "step"]
        assert steps[-1][1] % snapshot_every == 0 and not steps[-1][2]   # that step ran sequentially
    # with the snapshots taken out, the call sequence is the loop's without the hook
    assert [e for e in log if e != ("snapshot",)] == _run(max_steps, ingest_every, save_every)


def test_snapshot_interval_must_be_a_multiple_of_the_ingest_interval():
    from r2d2_b200.run_loop import run_learner_loop
    for bad in (0, -50, 25, 75):
        with pytest.raises(ValueError, match="snapshot_every"):
            run_learner_loop(None, None, max_steps=1, ingest_every=50, save_every=50, ingest=None, save=None,
                             snapshot=lambda: None, snapshot_every=bad)


# ---------------------------------------------------------------------------------------------- kernels
NEW_KERNELS = ("states_from_f16_kernel", "count_bad_leaves_kernel")


def test_restore_kernels_do_not_spill():
    report, stderr = ptxas_report("replay.cu")
    seen = set()
    for m in report:
        for k in NEW_KERNELS:
            if k in m.group(1):
                seen.add(k)
                assert m.group(2) == m.group(3) == m.group(4) == "0", m.group(0)
    assert seen == set(NEW_KERNELS), stderr[-2000:]


def test_restore_kernels_sass_has_no_local_memory():
    sass = library_sass()
    for k in NEW_KERNELS:
        funcs = functions(sass, k)
        assert len(funcs) == 1, (k, sorted(funcs))
        for name, body in funcs.items():
            body_ops = [op for op, _ in ops(body)]
            assert not [op for op in body_ops if op.startswith(("LDL", "STL"))], f"local-memory traffic in {name}"
    # the widening kernel moves 16 bytes per load
    body = next(iter(functions(sass, "states_from_f16_kernel").values()))
    assert any(op.startswith("LDG.E.128") for op, _ in ops(body))

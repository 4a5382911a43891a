"""Where global sampling's collectives sit in the learner's steps (tests/global_harness.py's global_schedule, built on
peer_schedule, which tests/test_cpu_peer_schedule.py holds to LearnerEngine.step), and run_loop's order around ingests.

The exchange buffers are single-buffered; their reuse is safe because of this order: every write-back (records
all-gather, then the filtered update) comes before the draw of the same hook or gap, the draw's three stages (root +
uniforms publish, draw + gather + delivery, delivery wait + weights) are consecutive, the pipelined draw fills the slot
the running iteration does not read, and the batch it fills is read (target or critic phase) only after the delivery
wait.  Nothing is drawn ahead of an ingest."""
import pytest

from global_harness import DRAW, WRITE_BACK, global_schedule
from r2d2_b200.run_loop import run_learner_loop


@pytest.mark.parametrize("prefetch", [False, True])
@pytest.mark.parametrize("target_interval", [1, 3, 500])
def test_write_back_then_draw_and_slot_reads_after_delivery(prefetch, target_interval):
    steps = 7
    sched = global_schedule(steps, target_interval, prefetch)
    flat = [c for step in sched for c in step]
    draws = [i for i, c in enumerate(flat) if c == ("draw", 0)]
    wbs = [i for i, c in enumerate(flat) if c == ("write_back", 0)]
    assert len(draws) == steps + (1 if prefetch else 0) - (0 if prefetch else 0)
    assert len(wbs) == len(draws) - 1                         # every draw after the first follows one write-back
    fill, lib = 0, 0
    for i, c in enumerate(flat):
        if c == ("draw", 0):
            assert flat[i:i + 3] == DRAW                      # the three stages back to back
            if i != draws[0]:
                j = max(w for w in wbs if w < i)
                assert flat[j:j + 2] == WRITE_BACK            # the write-back's two stages, before this draw
                between = flat[j + 2:i]
                assert between in ([], [("next_slot",)]), between
                assert not any(d for d in draws if j < d < i)
            if prefetch and i != draws[0]:
                assert fill != lib                            # the pipelined draw fills the slot not being trained
        if c == ("next_slot",):
            fill = 1 - fill
        if c[0] == "select_batch":
            lib = c[1]
        if c[0] in ("critic_phase", "target_phase"):
            slot = lib if c[0] == "critic_phase" else c[1]
            last_draw = max(d for d in draws if d < i)
            assert flat[last_draw + 2] == ("draw", 2) and last_draw + 2 < i
            if c[0] == "target_phase":
                assert slot == fill                           # the batch just delivered
        if c[0] == "critic_phase":
            assert slot == fill if not prefetch else lib == fill


class _Eng:
    def __init__(self, log):
        self.log, self.leaf_idx, self.priority = log, "leaf", "prio"

    def step(self, prefetch=None):
        self.log.append("step")
        if prefetch is not None:
            prefetch(self, self)


class _Replay:
    def __init__(self, log):
        self.log = log

    def update_priorities(self, leaf, prio):
        self.log.append("write_back")

    def sample_into(self, eng):
        self.log.append("draw")


@pytest.mark.parametrize("ingest_every", [1, 2, 3])
def test_run_loop_alternates_and_draws_nothing_ahead_of_an_ingest(ingest_every):
    log = []
    run_learner_loop(_Eng(log), _Replay(log), max_steps=7, ingest_every=ingest_every, save_every=100,
                     ingest=lambda: log.append("ingest"), save=lambda: None)
    seq = [x for x in log if x in ("write_back", "draw")]
    assert seq[0] == "draw" and all(a != b for a, b in zip(seq, seq[1:])), seq   # one write-back between two draws
    for i, x in enumerate(log):
        if x == "ingest":
            j = max(k for k in range(i) if log[k] in ("write_back", "draw"))
            assert log[j] == "write_back", log                 # the batch before an ingest is written back, none drawn

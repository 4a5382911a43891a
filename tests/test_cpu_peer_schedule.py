"""The call sequence of LearnerEngine.step / flush in the data-parallel "peer" mode is tests/peer_harness.peer_schedule.

The GPU exchange tests drive the phases group by group from peer_schedule instead of calling step(), so a change to the
order step() issues its phases in (a dropped early flush, a target chain run ahead of a target update, a moved hook)
has to fail here.  The engine runs on a recording stand-in for the library: no device is needed."""
from types import SimpleNamespace

import pytest

from peer_harness import peer_schedule

STEPS = 7


class _RecordingLib:
    """The learner entry points step() and flush() call; the step counter advances with each finish phase."""

    def __init__(self, log):
        self.log, self.count = log, 0

    def r2d2_learner_step_count(self, h):
        return self.count

    def r2d2_learner_select_batch(self, h, slot):
        self.log.append(("select_batch", slot))
        return 0

    def r2d2_learner_critic_phase(self, h, st):
        self.log.append(("critic_phase",))
        return 0

    def r2d2_learner_target_phase(self, h, slot, st):
        self.log.append(("target_phase", slot))
        return 0

    def r2d2_learner_actor_forward(self, h, st):
        self.log.append(("actor_forward",))
        return 0

    def r2d2_learner_actor_phase(self, h, scale, st):
        self.log.append(("actor_phase",))
        self.scales.append(scale)
        return 0

    def r2d2_learner_finish_phase(self, h, scale, st):
        self.log.append(("finish_phase",))
        self.scales.append(scale)
        self.count += 1
        return 0

    scales = None


def _engine(monkeypatch, world, target_interval):
    from r2d2_b200 import engine as E
    from r2d2_b200 import native as nv
    monkeypatch.setattr(nv, "current_stream", lambda: "stream")
    log = []
    lib = _RecordingLib(log)
    lib.scales = []
    eng = object.__new__(E.LearnerEngine)
    eng.lib, eng._h = lib, "handle"
    eng.cfg = E.PathConfig(obs=3, act=2, target_interval=target_interval)
    eng.world, eng._dist, eng._dp_mode = world, SimpleNamespace(), "peer"
    eng._pending_finish, eng._targets_ahead = False, False
    eng._slots = [{"leaf_idx": ("leaf", s), "is_weight": ("w", s)} for s in (0, 1)]
    eng.priority, eng.losses = "priority", "losses"
    eng._lib_slot = 0
    eng._bind_slot(0)
    return eng, log, lib


@pytest.mark.parametrize("world", [2, 5])
@pytest.mark.parametrize("prefetch", [False, True])
@pytest.mark.parametrize("target_interval", [1, 3, 500])
def test_step_issues_the_peer_schedule(monkeypatch, world, prefetch, target_interval):
    eng, log, lib = _engine(monkeypatch, world, target_interval)

    def hook(e, used):
        assert used.leaf_idx == ("leaf", 1 - e._fill_slot)       # the slot just trained on
        log.append(("prefetch",))

    got = []
    for _ in range(STEPS):
        eng.step(prefetch=hook if prefetch else None)
        got.append(log[:])
        log.clear()
    eng.flush()
    got.append(log[:])
    want = peer_schedule(STEPS, target_interval, prefetch)
    assert got == want
    assert lib.count == STEPS
    assert lib.scales == [1.0 / world] * (2 * STEPS)


def test_schedule_has_the_early_flushes_and_the_run_ahead_target_chains():
    """What the sequences above hold, spelled out: at interval 3 the finish phases of iterations 3 and 6 (the target
    updates) run before the next critic phase, and only the other iterations run the next batch's target chains ahead."""
    s = peer_schedule(STEPS, 3, True)
    early = [i for i, c in enumerate(s[:-1]) if c.index(("critic_phase",)) > 0 and ("finish_phase",) in c[:c.index(("critic_phase",))]]
    assert early == [3, 6]
    ahead = [i for i, c in enumerate(s[:-1]) if any(x[0] == "target_phase" for x in c)]
    assert ahead == [0, 1, 3, 4, 6]
    assert s[-1] == [("finish_phase",)]
    assert sum(c.count(("finish_phase",)) for c in s) == STEPS
    assert not any(x[0] == "target_phase" for c in peer_schedule(STEPS, 1, True) for x in c)   # every one updates
    assert not any(("finish_phase",) in c[:c.index(("critic_phase",))] for c in peer_schedule(STEPS, 500, False)[:-1])

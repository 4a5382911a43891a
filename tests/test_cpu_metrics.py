"""Learner metrics on the CPU (r2d2_b200.metrics): the environment switch, the CSV writer, the read rule of
LearnerMetrics against a host stand-in of the device ring, and the drop-in learner's log points on a fake engine."""
import csv
import math
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from learner_harness import fake_engine_learner
from r2d2_b200 import metrics as M


def test_environment_switch():
    assert M.from_environ({}) is False
    assert M.from_environ({"R2D2_METRICS": "0"}) is False
    assert M.from_environ({"R2D2_METRICS": "1"}) is True
    for bad in ("", "yes", "2", "true"):
        with pytest.raises(ValueError, match="R2D2_METRICS=.*allowed values are 0, 1"):
            M.from_environ({"R2D2_METRICS": bad})


def test_library_names_the_fields():
    from r2d2_b200 import native as nv
    lib = nv.lib()
    names = M.field_names()
    assert len(names) == lib.r2d2_metrics_field_count() == 23
    assert names[0] == "iteration" and names[21] == "actor_grad_norm" and names[-1] == "nonfinite"
    assert lib.r2d2_metrics_field_name(23) is None and lib.r2d2_metrics_field_name(-1) is None
    assert lib.r2d2_metrics_ring_bytes(1024) == 1024 * (23 * 8 + 4) and lib.r2d2_metrics_ring_bytes(0) == 0


def _rows(path):
    with open(path) as f:
        return list(csv.reader(f))


def test_csv_header_once_and_appends_across_a_resume(tmp_path):
    path = str(tmp_path / "metrics" / "x.csv")
    M.append_csv(path, ("a", "b"), [])
    assert not os.path.exists(path)                       # nothing to write: no file
    M.append_csv(path, ("a", "b"), [(1, 0.1), (2, float("nan"))])
    M.append_csv(path, ("a", "b"), [(3, True)])           # a resumed run appends to the same file
    rows = _rows(path)
    assert rows[0] == ["a", "b"] and len(rows) == 4
    assert float(rows[1][1]) == 0.1 and math.isnan(float(rows[2][1])) and rows[3] == ["3", "1"]


class _Ring:
    """Host stand-in of a learner and its metrics ring: critic(i) writes record i, finish(i) its actor norm and the step
    count, as the library does."""

    def __init__(self, slots):
        self.names = M.field_names()
        self.slots = slots
        self.records = np.full((slots, len(self.names)), np.nan)
        self.norms = np.full(slots, np.nan, np.float32)
        self.done = 0
        self.fetches = 0

    def critic(self, i):
        r = self.records[i % self.slots]
        r[:] = i + 0.25
        r[0] = i
        r[21] = np.nan

    def finish(self, i):
        assert i == self.done
        self.norms[i % self.slots] = i + 0.5
        self.done += 1

    def fetch(self):
        self.fetches += 1
        return self.records.copy(), self.norms.copy()

    def reader(self, first=0):
        return M.LearnerMetrics(lambda: self.done, self.fetch, self.names, self.slots, first)


def test_records_appear_after_their_finish_phase():
    ring = _Ring(8)
    m = ring.reader()
    ring.critic(0)
    assert m.read()["iteration"].size == 0 and ring.fetches == 0     # nothing finished: no copy at all
    ring.finish(0)
    ring.critic(1)
    ring.finish(1)
    out = m.read()
    assert out["iteration"].tolist() == [0, 1] and out["actor_grad_norm"].tolist() == [0.5, 1.5]
    assert out["q_mean"].tolist() == [0.25, 1.25]
    assert m.read()["iteration"].size == 0                             # each iteration is returned once


def test_deferred_finish_appears_one_read_later():
    ring = _Ring(8)
    m = ring.reader(first=40)                                          # a resumed run: numbering from the step count
    ring.done = 40
    ring.critic(40)                                                    # data parallel: finish(i) follows critic(i + 1)
    assert m.read()["iteration"].size == 0
    ring.critic(41)
    ring.finish(40)
    assert m.read()["iteration"].tolist() == [40]
    ring.finish(41)
    out = m.read()
    assert out["iteration"].tolist() == [41] and out["actor_grad_norm"].tolist() == [41.5]


def test_overrun_raises_naming_both_iterations():
    ring = _Ring(4)
    m = ring.reader()
    for i in range(6):
        ring.critic(i)
        ring.finish(i)
    with pytest.raises(RuntimeError, match="iteration 4 overwrote iteration 0"):
        m.read()


class _MetricsEngine:
    """What Learner.run touches of a LearnerEngine, with a metrics reader over a _Ring."""

    def __init__(self, cfg):
        self.cfg, self.device = cfg, None
        self.ring = _Ring(M.SLOTS)
        self.metrics = self.ring.reader()
        self.leaf_idx = self.priority = None

    def step(self, prefetch=None):
        i = self.ring.done
        self.ring.critic(i)
        self.ring.finish(i)
        if prefetch is not None:
            prefetch(self, SimpleNamespace(leaf_idx=None, priority=None))

    def views(self, net):
        return {}

    def enable_data_parallel(self):
        pass


def test_dropin_learner_logs_at_log_points_and_at_the_end(monkeypatch, tmp_path, capsys):
    lr = fake_engine_learner(monkeypatch, tmp_path, R2D2_METRICS="1", R2D2_SAVE_STATE="0")
    assert lr.engine.cfg.metrics is True
    lr.engine = _MetricsEngine(lr.engine.cfg)
    replay = SimpleNamespace(sample_into=lambda eng: None, update_priorities=lambda leaf, prio: None)
    lr.memory = SimpleNamespace(sequence_counter=10 ** 9, _dev=replay)
    seen = []
    read = lr.engine.metrics.read

    def counting_read():
        out = read()
        seen.append(out["iteration"].tolist())
        return out
    lr.engine.metrics.read = counting_read
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a: None)    # run() ends with one; no device here
    lr.run(max_steps=250)
    # log points before steps 0, 100 and 200, then the end of the run
    assert [(s[0], s[-1]) if s else None for s in seen] == [None, (0, 99), (100, 199), (200, 249)]
    rows = _rows("model_data/metrics/learner_rank0.csv")
    assert rows[0] == list(M.field_names()) and len(rows) == 251
    assert [int(r[0]) for r in rows[1:]] == list(range(250))
    assert float(rows[1][21]) == 0.5                                   # actor_grad_norm: the widened side array
    out = capsys.readouterr().out.splitlines()
    i = out.index("learning step: 100")
    assert out[i + 1].startswith("metrics: iterations 0-99 critic_loss")
    assert out[-1].startswith("metrics: iterations 200-249")


def test_dropin_learner_without_metrics_writes_nothing(monkeypatch, tmp_path):
    lr = fake_engine_learner(monkeypatch, tmp_path)
    assert lr.engine.cfg.metrics is False
    lr.log_metrics()
    assert not os.path.exists("model_data/metrics")

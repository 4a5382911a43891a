"""Learner metrics and episode returns: what a run reports about its training, off by default.

R2D2_METRICS=0|1 (default 0; any other value raises).  On:

  * the library reduces one record per learner iteration on the device, in the learner's stream, into a ring of
    `SLOTS` records (include/r2d2_b200.h, r2d2_learner_set_metrics: losses, Q / target / |TD error| / priority /
    importance-weight statistics, actor saturation, both gradient norms, a count of non-finite values).  The field names
    come from the library, the one place that knows the record format.
  * `LearnerMetrics.read()` returns the records of every iteration whose finish phase has been issued and that no
    earlier read returned, in iteration order: one device-to-host copy of the ring and one stream synchronisation, the
    only synchronisation the feature adds.  A data-parallel finish phase that is still deferred behind the next critic
    phase shows up in the next read; read() never completes it.  A wanted slot that already holds a later iteration
    means the ring overran (more than SLOTS iterations between two reads): read() raises.
  * the drop-in learner appends the records to ./model_data/metrics/learner_rank{r}.csv at each of its log points and
    when run() returns; the drop-in Actor and ActorPool append one row per finished episode to
    ./model_data/metrics/episodes_actor{id}.csv / episodes_pool{first id}.csv.  Both use `append_csv`.
"""
from __future__ import annotations

import csv
import os

import numpy as np

ENV = "R2D2_METRICS"
SLOTS = 1024          # records in the device ring: ten log intervals of 100 steps
METRICS_DIR = "./model_data/metrics/"
EPISODE_COLUMNS = ("actor_id", "episode", "step", "length", "return", "kept")
# the fields of the learner's summary line (means over the log interval; nonfinite is summed)
SUMMARY = ("critic_loss", "actor_loss", "q_mean", "target_mean", "td_abs_mean", "priority_mean", "mu_abs_mean",
           "mu_saturated", "critic_grad_norm", "actor_grad_norm")


def from_environ(env=None) -> bool:
    """R2D2_METRICS=0|1 (default 0)."""
    v = (os.environ if env is None else env).get(ENV, "0")
    if v not in ("0", "1"):
        raise ValueError("%s=%r: allowed values are 0, 1" % (ENV, v))
    return v == "1"


_names = None


def field_names() -> tuple:
    """The record's field names, in order, as the library reports them."""
    global _names
    if _names is None:
        from . import native as nv
        lib = nv.lib()
        _names = tuple(lib.r2d2_metrics_field_name(k).decode() for k in range(lib.r2d2_metrics_field_count()))
    return _names


def _cell(v) -> str:
    if isinstance(v, (bool, np.bool_)):
        return str(int(v))
    if isinstance(v, (int, np.integer)):
        return str(int(v))
    return "%.17g" % float(v)      # round-trips a double; integral values print without a fraction


def append_csv(path: str, columns, rows) -> None:
    """Append `rows` (sequences in the order of `columns`) to the CSV file at `path`, writing the header row first when
    the file is new or empty; the directory is created if needed.  Appending to an existing file (a resumed run) adds
    rows only."""
    rows = list(rows)
    if not rows:
        return
    d = os.path.dirname(path)
    if d:
        os.makedirs(d, exist_ok=True)
    new = not os.path.isfile(path) or os.path.getsize(path) == 0
    with open(path, "a", newline="") as f:
        w = csv.writer(f)
        if new:
            w.writerow(columns)
        for r in rows:
            w.writerow([_cell(v) for v in r])


def append_records(path: str, records: dict) -> None:
    """One CSV row per iteration of a read() result."""
    cols = list(records)
    append_csv(path, cols, zip(*(records[c] for c in cols)))


def summary_line(records: dict) -> str:
    """One line: the interval's iterations, the means of SUMMARY and the total non-finite count."""
    it = records["iteration"]
    parts = ["metrics: iterations %d-%d" % (int(it[0]), int(it[-1]))]
    parts += ["%s %.4g" % (k, float(np.mean(records[k]))) for k in SUMMARY]
    parts.append("nonfinite %d" % int(np.sum(records["nonfinite"])))
    return " ".join(parts)


def episode_csv(kind: str, actor_id: int) -> str:
    """./model_data/metrics/episodes_{kind}{actor_id}.csv (kind "actor" or "pool")."""
    return os.path.join(METRICS_DIR, "episodes_%s%d.csv" % (kind, actor_id))


class LearnerMetrics:
    """Reader of a learner's metrics ring.  `finished()` gives the number of finish phases issued (the library's step
    count), `fetch()` one host copy of the ring as (records [slots, F] float64, actor norms [slots] float32); `first`
    is the first iteration to return.  `attach(engine)` builds one on a LearnerEngine; tests pass fakes."""

    def __init__(self, finished, fetch, names, slots: int, first: int = 0):
        self._finished, self._fetch = finished, fetch
        self.names, self.slots, self.next = tuple(names), int(slots), int(first)

    @classmethod
    def attach(cls, engine, slots: int = SLOTS):
        """Allocate the ring on the engine's device and hand it to the library (before the engine's first step).
        `slots` is SLOTS for every engine; tests pass small rings to reach an overrun."""
        import torch

        from . import native as nv
        names = field_names()
        F = len(names)
        lib, h = engine.lib, engine._h
        ring = torch.full((slots * F + (slots + 1) // 2,), float("nan"), dtype=torch.float64, device=engine.device)
        assert ring.numel() * 8 >= int(lib.r2d2_metrics_ring_bytes(slots))
        nv.check(lib.r2d2_learner_set_metrics(h, nv.dptr(ring, torch.float64), int(slots)))

        def fetch():
            host = ring.cpu()                       # one D2H copy on the learner's stream, then a synchronisation
            return (host[:slots * F].numpy().reshape(slots, F),
                    host.view(torch.float32)[2 * slots * F:2 * slots * F + slots].numpy())

        m = cls(lambda: int(lib.r2d2_learner_step_count(h)), fetch, names, slots,
                int(lib.r2d2_learner_step_count(h)))
        m.ring = ring
        return m

    def read(self) -> dict:
        """{name: float64 array} of the iterations finished since the last read, in iteration order (empty arrays when
        there are none).  actor_grad_norm is the finish phase's float norm widened."""
        done = self._finished()
        if done <= self.next:
            return {n: np.zeros(0) for n in self.names}
        records, actor_norms = self._fetch()
        its = np.arange(self.next, done)
        rows = its % self.slots
        owner = records[rows, 0]
        bad = np.flatnonzero(owner != its)
        if bad.size:
            want, got = int(its[bad[0]]), owner[bad[0]]
            if np.isfinite(got) and got > want:
                raise RuntimeError("learner metrics ring of %d slots overran: iteration %d overwrote iteration %d before "
                                   "it was read (read at least every %d iterations)"
                                   % (self.slots, int(got), want, self.slots))
            raise RuntimeError("learner metrics: slot %d holds iteration %r, not the finished iteration %d"
                               % (want % self.slots, got, want))
        out = {n: records[rows, k].copy() for k, n in enumerate(self.names)}
        out["actor_grad_norm"] = actor_norms[rows].astype(np.float64)
        self.next = done
        return out

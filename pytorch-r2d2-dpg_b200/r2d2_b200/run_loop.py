"""The learner's training loop (learner.py:77-149 of the reference) as pure host logic: which call follows which.

    reference, per step:   sample -> iteration -> priority write-back -> [save] -> [ingest actor files]

Here the write-back of batch i and the draw of batch i+1 are handed to `engine.step(prefetch=...)`, which calls them as
soon as the priorities of batch i exist and runs the target chains of batch i+1 in the middle of iteration i (DESIGN
section 4).  Two rules keep the data the same as in the sequential loop:

  * priorities of batch i are written back before batch i+1 is drawn (always, it is the same hook);
  * nothing is drawn ahead of an ingest: an ingest may evict rows, and a batch drawn before it would later write its
    priorities onto rows that belong to other episodes by then.  The step in front of an ingest (and the last step of a
    bounded run) is sequential.

Global sampling (PathConfig.global_sampling) relies on both rules and on one more fact of this loop: every rank runs the
same steps, so every rank ingests on the same steps.  Its write-back and draw are collectives over the ranks' shards;
with nothing drawn ahead of an ingest and the ingests in step, each shard publishes its root after its own write-back
and ingest, and no rank's draw can meet rows a peer's ingest is still replacing.

Replay snapshots (`snapshot`, every `snapshot_every` steps, a multiple of `ingest_every`) are taken right after the
ingest of their step.  That step ran sequentially, so no batch is prefetched and no write-back is pending: the shard,
the nets and the RNG that draws the next batch are all at the same point.

Observation normalisation (`exchange`, PathConfig.obs_norm): the statistics the gathers read change only at
`exchange()`, a collective over the data-parallel ranks.  The loop calls it once before its first step and after every
ingest (before that step's snapshot): every rank runs the same steps, so every rank makes the same number of calls, and
since nothing is drawn ahead of an ingest, a pipelined, a sequential and a resumed run see the same statistics on every
batch.  The warm-up ingests before the loop (`warm_up`) stay local: the warm-up gate is per rank and passes after a
different number of ingests on each.

No CUDA, no torch: `engine` needs step(prefetch=None) + leaf_idx / priority attributes, `replay` needs sample_into(engine)
and update_priorities(leaf_idx, priority) - tests drive it with recording fakes (tests/test_cpu_host.py).
"""
from __future__ import annotations


def warm_up(ingest, ready, pause=None, report=None) -> int:
    """The warm-up gate (learner.py:69-75): `ingest()` until `ready()`, with `pause()` and `report()` after each.  Makes
    no collective call.  Returns the number of ingests."""
    n = 0
    while not ready():
        ingest()
        n += 1
        if pause is not None:
            pause()
        if report is not None:
            report()
    return n


def run_learner_loop(engine, replay, *, max_steps=None, ingest_every: int, save_every: int, ingest, save,
                     log=None, log_every: int = 100, snapshot=None, snapshot_every: int = 0, exchange=None) -> int:
    """Returns the number of steps run.  `ingest()` / `save()` are called after the steps whose number is a multiple of
    `ingest_every` / `save_every` (learner.py:141-149), `log(step)` before every `log_every`-th step (learner.py:79-80),
    `snapshot()`, if given, after the ingest of every `snapshot_every`-th step, and `exchange()`, if given, before the
    first step and right after every ingest."""
    if ingest_every < 1 or save_every < 1:
        raise ValueError("ingest_every and save_every must be >= 1")
    if snapshot is not None and (snapshot_every < 1 or snapshot_every % ingest_every):
        raise ValueError("snapshot_every must be a positive multiple of ingest_every (%d), got %r"
                         % (ingest_every, snapshot_every))

    def next_batch(eng, used):
        replay.update_priorities(used.leaf_idx, used.priority)      # learner.py:135-139
        replay.sample_into(eng)                                     # learner.py:84 of the next iteration

    step = 0
    have_batch = False
    if exchange is not None:
        exchange()
    while max_steps is None or step < max_steps:
        if log is not None and step % log_every == 0:
            log(step)
        step += 1
        if not have_batch:
            replay.sample_into(engine)                              # learner.py:84
        if step % ingest_every == 0 or step == max_steps:
            engine.step()                                           # learner.py:86-132
            replay.update_priorities(engine.leaf_idx, engine.priority)
            have_batch = False
        else:
            engine.step(prefetch=next_batch)
            have_batch = True
        if step % save_every == 0:
            save()
        if step % ingest_every == 0:
            ingest()                                                # learner.py:144-149 without the sleep stall
            if exchange is not None:
                exchange()
            if snapshot is not None and step % snapshot_every == 0:
                snapshot()
    return step

"""Concurrent chains (csrc/learner.cu, learner_critic_phase): on one GPU the actor's forward chain runs on the learner's
aux stream beside the online critic's, and the critic BPTT beside the next batch's target chains.  Every kernel computes
what it computes in the serial order, so the schedule must not change a bit:

 (a) replay-fed pipelined steps at cfg-3's H = 512, B = 512 across a target update, default schedule against
     R2D2_OVERLAP_INPUTS=0 (the fully serial order) in separate engines: per iteration q, target, priorities and
     losses, then both nets, their targets and Adam moments; also with the twin critic and the metrics ring on;
 (b) two in-process data-parallel ranks (tests/peer_harness.py), which keep the serial order, under both settings."""
import numpy as np
import pytest
import torch

from learner_harness import assert_same_bits, episode, snapshot
from oracle import ref_port
from peer_harness import PeerGroup, split_batch

pytestmark = pytest.mark.gpu

CFG3 = dict(obs=376, act=17, hidden=512, batch=512, burn_in=40, learning=80, n_step=5)
STEPS = 7                      # target interval 4: the 4th iteration updates the targets, so its hook runs last
OPTIONS = {"defaults": {}, "twin_metrics": dict(twin_critic=True, metrics=True)}


@pytest.fixture(scope="module")
def E():
    from r2d2_b200 import engine
    engine.nv.lib()
    return engine


def _replay_fed(E, monkeypatch, serial, extra):
    """Per-iteration outputs and the final snapshot of STEPS pipelined iterations fed from a seeded replay shard."""
    if serial:
        monkeypatch.setenv("R2D2_OVERLAP_INPUTS", "0")
    else:
        monkeypatch.delenv("R2D2_OVERLAP_INPUTS", raising=False)
    cfg = E.PathConfig(**CFG3, target_interval=4, **extra)
    rng = np.random.default_rng(3)
    rp = E.DeviceReplay(cfg, capacity_rows=12 * (250 + cfg.n_step))
    rp.add_episodes([episode(rng, cfg, 250) for _ in range(12)])
    eng = E.LearnerEngine(cfg, seed=5)
    gen = torch.Generator(device="cuda").manual_seed(17)

    def hook(e, used):
        rp.update_priorities(used.leaf_idx, used.priority)
        rp.sample_into(e, generator=gen)

    per_it = []
    rp.sample_into(eng, generator=gen)
    for _ in range(STEPS):
        eng.step(prefetch=hook)
        keys = ["q_value", "target_q_value", "priority", "losses"] + (["q_value2"] if cfg.twin_critic else [])
        per_it.append({k: getattr(eng, k).clone() for k in keys})
    out = snapshot(eng)
    if eng.metrics is not None:   # every record but its %globaltimer stamp, and the actor norms; bits (NaN-filled slots)
        m = eng.metrics
        F = len(m.names)
        rec = m.ring[:m.slots * F].view(m.slots, F).clone()
        rec[:, m.names.index("t_ns")] = 0
        out["metrics_records"] = rec.view(torch.int64)
        out["metrics_actor_norms"] = m.ring[m.slots * F:].view(torch.int64).clone()
        assert int((rec[:, 0] == rec[:, 0]).sum()) == STEPS   # one record per iteration
    out["launches"] = torch.tensor(eng.launches_per_iteration)
    torch.cuda.synchronize()
    rp.close()
    eng.close()
    return per_it, out


@pytest.mark.parametrize("option", sorted(OPTIONS))
def test_concurrent_chains_match_the_serial_order_at_cfg3(E, monkeypatch, option):
    serial_it, serial = _replay_fed(E, monkeypatch, True, OPTIONS[option])
    conc_it, conc = _replay_fed(E, monkeypatch, False, OPTIONS[option])
    for it, (a, b) in enumerate(zip(serial_it, conc_it)):
        for k in a:
            assert torch.equal(a[k], b[k]), f"iteration {it}: {k}"
    assert_same_bits(serial, conc)


SMALL = dict(obs=6, act=2, hidden=64, batch=8, burn_in=4, learning=6, n_step=2)


def _two_ranks(monkeypatch, serial, shards):
    if serial:
        monkeypatch.setenv("R2D2_OVERLAP_INPUTS", "0")
    else:
        monkeypatch.delenv("R2D2_OVERLAP_INPUTS", raising=False)
    g = PeerGroup(2, dict(SMALL, target_interval=3))
    try:
        g.run(shards, prefetch=True)
        g.check_status()
        out = [{k: v.clone() for k, v in snapshot(eng).items()} for eng in g.engines]
    finally:
        g.close()
    return out


def test_two_ranks_are_the_same_under_both_settings(E, monkeypatch):
    pc = ref_port.PathConfig(**dict(SMALL, batch=2 * SMALL["batch"]))
    shards = [split_batch(ref_port.synthetic_batch(pc, seed=90 + i), 2) for i in range(STEPS + 1)]
    serial = _two_ranks(monkeypatch, True, shards)
    conc = _two_ranks(monkeypatch, False, shards)
    for r in range(2):
        assert_same_bits(serial[r], conc[r])

"""CPU-only checks: the C-ABI library loads and exports every symbol include/r2d2_b200.h declares, the
sum-tree oracle behaves, the drop-in host modules keep the reference's formats, and the data-parallel
decomposition (mean of per-rank gradients == global-batch gradient) holds under a world_size-2 gloo run."""
import os
import re
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from conftest import PKG, ROOT, load_golden
from oracle import learner_oracle as lo
from oracle import ref_port
from oracle.sumtree import SumTreeOracle


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "r2d2_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(r2d2_[a-z0-9_]+)\s*\(", text)))


def test_abi_exports_every_declared_symbol():
    from r2d2_b200 import native
    lib_path = native.LIB_PATH
    assert os.path.isfile(lib_path), "run __graft_entry__.build() first"
    exported = set(re.findall(r" T (r2d2_[a-z0-9_]+)", subprocess.check_output(["nm", "-D", lib_path], text=True)))
    declared = _declared_symbols()
    assert declared, "header parse failed"
    missing = [s for s in declared if s not in exported]
    assert not missing, f"declared but not exported: {missing}"
    unbound = [s for s in declared if s not in native.SIGNATURES]
    assert not unbound, f"declared but not bound in native.SIGNATURES: {unbound}"
    lib = native.lib()                       # loads, resolves every symbol (no GPU needed)
    assert lib.r2d2_arch() == b"sm_90a" and lib.r2d2_version() >= 100


def test_no_cpu_fallback():
    from r2d2_b200 import engine, native
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(native.NativeError):
        engine.LearnerEngine(engine.PathConfig(obs=3, act=1))
    with pytest.raises(native.NativeError):
        engine.DeviceReplay(engine.PathConfig(obs=3, act=1), capacity_rows=128)


def test_sass_is_hopper_native():
    """The shipped binary is sm_90a code with wgmma (HGMMA), bulk copies (UBLKCP) and mbarrier waits (SYNCS)."""
    from r2d2_b200 import native
    sass = subprocess.run(["cuobjdump", "-sass", native.LIB_PATH], capture_output=True, text=True).stdout
    if not sass:
        pytest.skip("cuobjdump unavailable")
    assert "arch = sm_90a" in sass
    for mnemonic in ("HGMMA", "UBLKCP", "SYNCS"):
        assert mnemonic in sass, mnemonic


# ---------------------------------------------------------------------------------------------- sum tree
def test_sumtree_oracle_edges():
    t = SumTreeOracle(1000)
    assert t.sample(np.float32([0.0, 0.5]))[0] == 0            # empty tree: index 0
    p = np.zeros(1000, np.float32)
    p[[3, 500, 999]] = [1.0, 2.0, 1.0]
    t.set_range(0, p)
    assert t.total == 4.0
    u = np.float32([0.0, 0.2499, 0.25, 0.7499, 0.75, np.nextafter(np.float32(1), np.float32(0))])
    assert list(t.sample(u)) == [3, 3, 500, 500, 999, 999]
    t.update_batch([500, 500, 3], np.float32([5.0, 0.0, 1.0]))   # duplicates: last write wins
    assert t.total == 2.0 and set(t.sample(np.random.default_rng(0).uniform(size=1000).astype(np.float32))) == {3, 999}


def test_sumtree_matches_reference_sampler_distribution():
    g = load_golden("ref_sampler_hist.npz")
    pri = g["priorities"].astype(np.float32)
    t = SumTreeOracle(len(pri))
    t.set_range(0, pri)
    n = 200000
    cnt = np.bincount(t.sample(np.random.default_rng(1).uniform(size=n).astype(np.float32)), minlength=len(pri))
    exp = pri.astype(np.float64) / pri.astype(np.float64).sum() * n
    assert 0.7 < ((cnt - exp) ** 2 / exp).sum() / len(pri) < 1.3
    exp_ref = pri.astype(np.float64) / pri.astype(np.float64).sum() * int(g["n_draws"])
    assert 0.7 < ((g["counts"] - exp_ref) ** 2 / exp_ref).sum() / len(pri) < 1.3


# ---------------------------------------------------------------------------------------------- drop-in host side
def test_dropin_utils_match_reference_kat():
    import utils as dropin_utils
    k = load_golden("ref_kat.npz")
    assert abs(dropin_utils.calc_priority(k["calc_priority_in"]) - float(k["calc_priority_out"])) < 1e-6
    assert np.allclose(dropin_utils.invertical_vf(torch.tensor(k["h_in"])).numpy(), k["h_out"], rtol=1e-6, atol=0)
    from collections import OrderedDict
    obs = dropin_utils.get_obs(OrderedDict(a=np.arange(3.0), b=2.5, c=np.ones(2)))
    assert obs.shape == (1, 6) and obs.dtype == np.float32 and list(obs[0]) == [0, 1, 2, 2.5, 1, 1]


def test_dropin_models_state_dict_layout_matches_flat_views():
    import models as dropin_models
    from r2d2_b200 import engine
    cfg = engine.PathConfig(obs=7, act=3, hidden=64)
    for critic, cls in ((False, dropin_models.ActorNet), (True, dropin_models.CriticNet)):
        net = cls(7, 3, 0, hidden=64)
        sd = net.state_dict()
        assert list(sd.keys()) == list(engine.PARAM_KEYS)
        assert {k: tuple(v.shape) for k, v in sd.items()} == dict(engine.param_shapes(cfg, critic))
        flat = torch.cat([v.reshape(-1) for v in sd.values()])
        for k, v in engine.flat_views(flat, cfg, critic).items():
            assert torch.equal(v, sd[k])


def test_actor_file_protocol_roundtrip(monkeypatch):
    """Synthetic actor -> memory0.pt in the reference format -> pack_episode (what the learner ingests)."""
    monkeypatch.setenv("R2D2_OBS_SIZE", "5")
    monkeypatch.setenv("R2D2_N_ACTIONS", "2")
    monkeypatch.setenv("R2D2_HIDDEN", "32")
    import actor as dropin_actor
    import replay_memory as dropin_rm
    with tempfile.TemporaryDirectory() as d:
        cwd = os.getcwd()
        os.chdir(d)
        try:
            os.makedirs("model_data")
            os.makedirs("memory_data")
            a = dropin_actor.Actor(0)
            a.env.episode_len = 66
            a.run(max_episodes=5)
            payload = torch.load("memory_data/memory0.pt", weights_only=False)
        finally:
            os.chdir(cwd)
    assert set(payload) == {"replay_memory", "recurrent_state", "priority", "total_priority"}
    rows, states, prio = payload["replay_memory"][0], payload["recurrent_state"][0], payload["priority"][0]
    assert len(rows) == 66 + 5 and len(states) == 66 and len(prio) == 66 - 60      # actor.py:106-107,173
    obs, act, rew, term, st = dropin_rm.pack_episode(rows, states, hidden=32)
    assert obs.shape == (71, 5) and act.shape == (71, 2) and st.shape == (66, 4, 2, 32)
    assert term[-5:].tolist() == [1.0] * 5 and not obs[-5:].any()
    assert abs(payload["total_priority"][0] - sum(prio)) < 1e-9


# ---------------------------------------------------------------------------------------------- data parallel
def _dp_worker(rank, world, port, out_dir):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    pc = ref_port.PathConfig(obs=4, act=2, hidden=8, batch=6, burn_in=3, learning=5, n_step=2)
    port_l = ref_port.PortLearner(pc, seed=7)
    sd = lambda m: {k: v.detach().numpy() for k, v in m.state_dict().items()}  # noqa: E731
    full = ref_port.synthetic_batch(pc, seed=3)
    shard = {k: v[:, rank * 3:(rank + 1) * 3] for k, v in full.items()}

    def allreduce_mean(_net, grads):
        for k in lo.PARAM_KEYS:
            t = torch.from_numpy(grads[k])
            dist.all_reduce(t)
            grads[k][...] = (t / world).numpy()

    ol = lo.OracleLearner(sd(port_l.actor), sd(port_l.critic), burn_in=3, learning=5, n_step=2)
    for _ in range(2):
        out = ol.iteration(shard, grad_hook=allreduce_mean)
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), **{f"a/{k}": v for k, v in out["actor_after"].items()},
             **{f"c/{k}": v for k, v in out["critic_after"].items()})
    if rank == 0:
        ref = lo.OracleLearner(sd(port_l.actor), sd(port_l.critic), burn_in=3, learning=5, n_step=2)
        for _ in range(2):
            o = ref.iteration(full)
        np.savez(os.path.join(out_dir, "full.npz"), **{f"a/{k}": v for k, v in o["actor_after"].items()},
                 **{f"c/{k}": v for k, v in o["critic_after"].items()})
    dist.destroy_process_group()


def test_data_parallel_gradient_mean_equals_global_batch():
    """SURVEY 8e: equal shards + all-reduce-mean of the two gradient sets reproduce the single-learner update
    (losses are means over L*B*A, learner.py:111,124).  world_size 2, gloo, CPU oracle as the learner."""
    import torch.multiprocessing as mp
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_dp_worker, args=(2, 29533 + os.getpid() % 200, d), nprocs=2, join=True)
        full = np.load(os.path.join(d, "full.npz"))
        r0, r1 = np.load(os.path.join(d, "rank0.npz")), np.load(os.path.join(d, "rank1.npz"))
        for k in full.files:
            assert np.allclose(r0[k], r1[k], rtol=0, atol=0), k             # replicas stay identical
            assert np.allclose(r0[k], full[k], rtol=1e-9, atol=1e-12), k   # and equal the global-batch learner


def test_peer_exchange_layout_is_aligned_and_disjoint():
    """Data-parallel gradient exchange buffer (csrc/peer.cuh): [flags | critic grads | actor grads | critic sums | actor
    sums]; every block padded so that each of `world` ranks owns a whole number of float4, 256-byte aligned, disjoint."""
    from ctypes import byref
    from r2d2_b200 import native
    lib = native.lib()
    n_critic, n_actor = 2311697, 1381393          # odd sizes on purpose
    for world in (2, 3, 4, 8, 16):
        lay = native.PeerLayout()
        native.check(lib.r2d2_peer_layout_for(n_critic, n_actor, world, byref(lay)))
        q = 4 * world
        pad_c, pad_a = -(-n_critic // q) * q, -(-n_actor // q) * q
        blocks = [(lay.off_critic_grads, pad_c), (lay.off_actor_grads, pad_a), (lay.off_critic_sums, pad_c),
                  (lay.off_actor_sums, pad_a)]
        end = 4096                                 # the flag area
        for off, n in blocks:
            assert off % 256 == 0 and off >= end
            end = off + 4 * n
        assert lay.bytes >= end and lay.bytes % 256 == 0
    lay = native.PeerLayout()
    assert lib.r2d2_peer_layout_for(n_critic, n_actor, 1, byref(lay)) != 0      # one rank has nothing to exchange
    assert lib.r2d2_peer_layout_for(n_critic, n_actor, 17, byref(lay)) != 0


class _FakeEngine:
    """Records what run_learner_loop does.  Mimics LearnerEngine.step: the prefetch hook runs once per step, after the
    priorities of the current batch exist; the attributes leaf_idx / priority describe the batch in the engine."""

    def __init__(self, log):
        self.log, self.batch, self.leaf_idx, self.priority = log, None, None, None

    def step(self, prefetch=None):
        assert self.batch is not None, "step without a batch"
        trained = self.batch
        self.log.append(("step", trained, prefetch is not None))
        self.leaf_idx, self.priority = ("leaf", trained), ("prio", trained)
        if prefetch is not None:
            from types import SimpleNamespace
            used = SimpleNamespace(leaf_idx=self.leaf_idx, priority=self.priority)
            self.batch = None
            prefetch(self, used)
        else:
            self.batch = ("consumed", trained)


class _FakeReplay:
    def __init__(self, log):
        self.log, self.draws = log, 0

    def sample_into(self, eng):
        self.draws += 1
        eng.batch = self.draws
        self.log.append(("draw", self.draws))

    def update_priorities(self, leaf_idx, priority):
        assert leaf_idx[1] == priority[1]
        self.log.append(("writeback", leaf_idx[1]))


@pytest.mark.parametrize("max_steps,ingest_every,save_every", [(23, 5, 4), (10, 1, 3), (7, 50, 50), (12, 4, 4)])
def test_run_loop_keeps_the_sequential_data_flow(max_steps, ingest_every, save_every):
    """Host logic of Learner.run (r2d2_b200/run_loop.py): every batch is trained on once, its priorities are written
    back exactly once and before the next draw, nothing is drawn ahead of an ingest, saves / ingests fall on the
    reference's steps (learner.py:141-149)."""
    from r2d2_b200.run_loop import run_learner_loop
    log = []
    eng, rp = _FakeEngine(log), _FakeReplay(log)
    n = run_learner_loop(eng, rp, max_steps=max_steps, ingest_every=ingest_every, save_every=save_every,
                         ingest=lambda: log.append(("ingest",)), save=lambda: log.append(("save",)),
                         log=lambda s: log.append(("log", s)), log_every=5)
    assert n == max_steps
    steps = [e for e in log if e[0] == "step"]
    assert [e[1] for e in steps] == list(range(1, max_steps + 1))            # batch k is trained on in step k, once
    assert [e[1] for e in log if e[0] == "writeback"] == list(range(1, max_steps + 1))
    assert [e[1] for e in log if e[0] == "draw"] == list(range(1, max_steps + 1))   # no batch drawn and dropped
    pos = {e: i for i, e in enumerate(log)}
    for k in range(1, max_steps):
        assert pos[("writeback", k)] < pos[("draw", k + 1)]                  # tree is up to date for the next draw
    # ingests: after the steps that are multiples of ingest_every, and no batch is in flight across them
    ingest_at = [i for i, e in enumerate(log) if e[0] == "ingest"]
    assert len(ingest_at) == max_steps // ingest_every
    for i in ingest_at:
        done = [e[1] for e in log[:i] if e[0] == "step"]
        assert done and done[-1] % ingest_every == 0
        drawn = [e[1] for e in log[:i] if e[0] == "draw"]
        assert drawn[-1] == done[-1], "a batch was drawn ahead of an ingest"
    assert len([e for e in log if e[0] == "save"]) == max_steps // save_every
    # the steps in front of an ingest and the last one are sequential, all others hand the hook to the engine
    for _, k, pipelined in steps:
        assert pipelined == (k % ingest_every != 0 and k != max_steps)
    assert [e[1] for e in log if e[0] == "log"] == list(range(0, max_steps, 5))


def test_bench_configs_are_the_baseline_configs():
    """bench.py measures BASELINE.json's metric on BASELINE.json's shapes: configs[1] / configs[2] are parsed from the
    baseline's own strings, the headline (default --config) is configs[2], and both arms print the same workload."""
    import json
    sys.path.insert(0, ROOT)
    import bench
    base = json.load(open(os.path.join(ROOT, "BASELINE.json")))
    assert bench.METRIC.split(" (")[0] in base["metric"]

    def shape(text):
        kv = dict(re.findall(r"(obs|act|hidden|seq_len|burn_in|batch)=(\d+)", text))
        return {k: int(v) for k, v in kv.items()}

    for name, idx in (("cfg2", 1), ("cfg3", 2)):
        want, have = shape(base["configs"][idx]), bench.CONFIGS[name]
        assert want["obs"] == have["obs"] and want["act"] == have["act"] and want["hidden"] == have["hidden"]
        assert want["batch"] == have["batch"] and want["seq_len"] == have["learning"]
        assert want.get("burn_in", have["burn_in"]) == have["burn_in"]
    src = open(os.path.join(ROOT, "bench.py")).read()
    assert re.search(r'add_argument\("--config", default="cfg3"', src)
    assert src.count("workload_string(name, c)") >= 2          # the GPU arm and the reference arm
    line = bench.workload_string("cfg3", bench.CONFIGS["cfg3"])
    assert line == "cfg3: obs=376 act=17 hidden=512 batch=512 burn_in=40 learning=80 n_step=5"

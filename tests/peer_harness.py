"""An in-process data-parallel group for the peer-memory gradient exchange (csrc/peer.cu) on one device.

The exchange kernels take plain device pointers, so W `LearnerEngine`s in one process, each with its own zeroed buffer of
`r2d2_learner_peer_layout(world).bytes` handed to `r2d2_learner_attach_peers`, form a W-rank world: the same signal /
slice-sum / wait kernels at the same places of the phases as across GPUs, without NVLink mappings or cross-device memory
ordering.

`peer_schedule` is the call sequence `LearnerEngine.step` / `flush` make in peer mode (tests/test_cpu_peer_schedule.py
holds it to the engine).  `PeerGroup.run` issues that sequence group by group: each call for every rank on the rank's
own stream, every stream recording an event, and every stream waiting for all W events before the next call.  Issued that
way every signal has executed before a slice sum that needs it runs, so no slice-sum kernel waits; the only kernel that can
wait is the single-warp `peer_wait` of a finish phase that runs its own slice sum (an early flush before a target update,
or the last flush), and it waits for the other ranks' slice sums of the same group.  Those finish phases launch the
slice sum, the wait, the norm and Adam kernels and the target copies, none of which allocates scratch (elementwise.cu's
`partials_scratch` is not on that path; `grad_norm` uses the learner's own arena), so nothing in such a group
synchronises the device.  `step()` itself is not used: it issues all phases of one rank at once, and a slice sum of up to
132 CTAs would then wait on SMs while the other ranks' scans wait for them.

Kernels of streams that share a hardware work queue start in the order they were issued, so a rank's Adam kernel queued
behind its waiting `peer_wait` would hold back another rank's slice sum queued after it.  Each rank stream needs a queue
of its own: the module asks for CUDA's maximum of 32 (CUDA_DEVICE_MAX_CONNECTIONS, read when the CUDA context is
created, which in a test session happens after collection has imported this module)."""
from __future__ import annotations

import os

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

from ctypes import byref, c_int, c_void_p  # noqa: E402

import numpy as np  # noqa: E402

from kernel_harness import scan_status  # noqa: E402

# one rank's calls: ("select_batch", slot), ("critic_phase",), ("finish_phase",), ("prefetch",), ("target_phase", slot),
# ("actor_forward",), ("actor_phase",)


def peer_schedule(steps: int, target_interval: int, prefetch: bool):
    """The calls one rank makes for `steps` calls of LearnerEngine.step (with a prefetch hook or without) followed by
    flush(), in the data-parallel "peer" mode, starting from a fresh engine (step counter 0, both slots 0): a list of
    `steps` + 1 lists, the calls of each step and then those of the flush."""
    out = []
    count, pending, fill, lib_slot = 0, False, 0, 0

    def updates_targets():       # LearnerEngine._finish_updates_targets at library step counter `count`
        return target_interval > 0 and (count + 1) % target_interval == 0

    for _ in range(steps):
        calls = []
        out.append(calls)
        if fill != lib_slot:
            calls.append(("select_batch", fill))
            lib_slot = fill
        if pending and updates_targets():
            calls.append(("finish_phase",))          # early flush: the next target chains read the updated targets
            count, pending = count + 1, False
        calls.append(("critic_phase",))
        if pending:
            calls.append(("finish_phase",))          # the deferred phase 3 of the previous iteration
            count, pending = count + 1, False
        ahead = prefetch and not updates_targets()
        if ahead:
            calls.append(("prefetch",))
            fill = 1 - fill
            calls.append(("target_phase", fill))
        calls.append(("actor_forward",))
        calls.append(("actor_phase",))
        pending = True
        if prefetch and not ahead:
            calls.append(("prefetch",))
            fill = 1 - fill
    out.append([("finish_phase",)] if pending else [])   # the last flush
    return out


def padded(n: int, world: int) -> int:
    q = 4 * world
    return -(-n // q) * q


def split_batch(batch: dict, world: int) -> list:
    """A time-major global batch split along the batch axis (axis 1) into `world` equal shards; `is_weight` [B] too."""
    B = batch["obs"].shape[1]
    assert B % world == 0, (B, world)
    b = B // world
    out = []
    for r in range(world):
        s = {k: np.ascontiguousarray(v[:, r * b:(r + 1) * b]) for k, v in batch.items() if k != "is_weight"}
        if "is_weight" in batch:
            s["is_weight"] = np.ascontiguousarray(np.asarray(batch["is_weight"]).reshape(-1)[r * b:(r + 1) * b])
        out.append(s)
    return out


class PeerGroup:
    """W engines on the current device with identical nets, targets and moments (what enable_data_parallel broadcasts),
    one stream each, attached to each other's exchange buffers."""

    def __init__(self, world: int, path_kwargs: dict, seed: int = 1):
        import torch
        from r2d2_b200 import engine as E
        from r2d2_b200 import native as nv
        self.torch, self.nv, self.world = torch, nv, world
        self.engines = [E.LearnerEngine(E.PathConfig(**path_kwargs), seed=seed) for _ in range(world)]
        self.streams = [torch.cuda.Stream() for _ in range(world)]
        e0 = self.engines[0]
        self.lib = e0.lib
        lay = nv.PeerLayout()
        nv.check(self.lib.r2d2_learner_peer_layout(e0._h, world, byref(lay)))
        self.layout = lay
        self.n = {"critic": e0.grads["critic"].numel(), "actor": e0.grads["actor"].numel()}
        self.padded = {k: padded(v, world) for k, v in self.n.items()}
        off = {("grads", "critic"): lay.off_critic_grads, ("grads", "actor"): lay.off_actor_grads,
               ("sums", "critic"): lay.off_critic_sums, ("sums", "actor"): lay.off_actor_sums}
        torch.cuda.synchronize()
        self.bufs = [torch.zeros(int(lay.bytes) // 4, dtype=torch.float32, device=e0.device) for _ in range(world)]
        torch.cuda.synchronize()
        ptrs = (c_void_p * world)(*[b.data_ptr() for b in self.bufs])
        # full padded views of each rank's blocks: {"grads"|"sums": {"critic"|"actor": tensor}}
        self.blocks = []
        for r, (eng, buf) in enumerate(zip(self.engines, self.bufs)):
            for net in ("actor", "critic", "target_actor", "target_critic"):
                assert eng.flat[net].equal(e0.flat[net])
            nv.check(self.lib.r2d2_learner_attach_peers(eng._h, r, world, ptrs))
            nv.check(self.lib.r2d2_learner_set_overlap_actor_inputs(eng._h, 0))
            v = {w: {net: buf[int(off[(w, net)]) // 4:int(off[(w, net)]) // 4 + self.padded[net]]
                     for net in ("critic", "actor")} for w in ("grads", "sums")}
            self.blocks.append(v)
            eng.grads = {net: v["grads"][net][:self.n[net]] for net in ("actor", "critic")}   # as _attach_peers does
            eng.world = world
        self._events = None
        self.pending = None          # iteration whose finish phase is still due
        self.closed = False

    # ---- issue -------------------------------------------------------------------------------------------------
    def _issue(self, fn):
        """fn(rank, engine, stream) for every rank on its own stream, after every rank's previous group."""
        torch = self.torch
        events = []
        for r, (eng, s) in enumerate(zip(self.engines, self.streams)):
            if self._events is not None:
                for ev in self._events:
                    s.wait_event(ev)
            with torch.cuda.stream(s):
                fn(r, eng, s)
            ev = torch.cuda.Event()
            ev.record(s)
            events.append(ev)
        self._events = events

    def _call(self, name, *args):
        nv = self.nv

        def fn(r, eng, s):
            st = c_void_p(s.cuda_stream)
            if name == "select_batch":
                nv.check(self.lib.r2d2_learner_select_batch(eng._h, args[0]))
                eng._lib_slot = args[0]
            elif name == "target_phase":
                nv.check(self.lib.r2d2_learner_target_phase(eng._h, args[0], st))
            elif name in ("actor_phase", "finish_phase"):
                nv.check(getattr(self.lib, "r2d2_learner_" + name)(eng._h, 1.0 / self.world, st))
            else:
                nv.check(getattr(self.lib, "r2d2_learner_" + name)(eng._h, st))
        self._issue(fn)

    def sync(self):
        self.torch.cuda.synchronize()

    def set_batches(self, shards):
        """Write one shard per rank into the engines' fill slots (device tensors: no host copy inside a group)."""
        def fn(r, eng, s):
            eng.set_batch(shards[r])
        self._issue(fn)

    def to_device(self, shards):
        dev = self.engines[0].device
        return [{k: self.torch.as_tensor(np.asarray(v, np.float32)).to(dev) for k, v in s.items()} for s in shards]

    def run(self, batches, prefetch=False, on_critic=None, on_iteration=None, on_finish=None, final_flush=True):
        """Train on `batches`, a list over iterations of per-rank shard lists (one more than iterations when prefetching:
        the hook of the last step draws it).  Callbacks, called with the iteration index between groups (the device
        synchronised): on_critic after the critic phase group, on_iteration after the actor-phase group, on_finish after
        the finish group that completes that iteration."""
        steps = len(batches) - (1 if prefetch else 0)
        dev = [self.to_device(b) for b in batches]
        it, drawn = -1, 0
        schedule = peer_schedule(steps, self.engines[0].cfg.target_interval, prefetch)
        calls = []
        for i, step_calls in enumerate(schedule[:-1]):
            if i == 0 or not prefetch:
                calls.append(("set_batch", i))                # the caller's set_batch before step()
            calls += step_calls
        if final_flush:
            calls += schedule[-1]
        for c in calls:
            name = c[0]
            if name == "set_batch":
                self.set_batches(dev[c[1]])
                continue
            if name == "critic_phase":
                it += 1
            if name == "prefetch":
                drawn += 1
                nxt = dev[drawn]

                def fn(r, eng, s, nxt=nxt):
                    eng._bind_slot(1 - eng._fill_slot)     # LearnerEngine._run_prefetch
                    eng.set_batch(nxt[r])
                self._issue(fn)
                continue
            self._call(*c)
            if name == "critic_phase" and on_critic is not None:
                self.sync()
                on_critic(it)
            if name == "actor_phase":
                self.pending = it
                if on_iteration is not None:
                    self.sync()
                    on_iteration(it)
            if name == "finish_phase":
                done, self.pending = self.pending, None
                if on_finish is not None:
                    self.sync()
                    on_finish(done)
        self.sync()

    def flush(self):
        """The last flush: completes a pending finish phase on every rank."""
        if self.pending is not None:
            self._call("finish_phase")
            self.pending = None
        self.sync()

    # ---- read back ---------------------------------------------------------------------------------------------
    def block(self, what: str, net: str, rank: int, pad: bool = False) -> np.ndarray:
        t = self.blocks[rank][what][net]
        return (t if pad else t[:self.n[net]]).cpu().numpy()

    def peer_status(self):
        out = []
        for eng, s in zip(self.engines, self.streams):
            st = c_int(0)
            self.nv.check(self.lib.r2d2_learner_peer_status(eng._h, byref(st), c_void_p(s.cuda_stream)))
            out.append(int(st.value))
        return out

    def scan_status(self):
        """The scans' device-wide flag (sticky until read): 1 when a bounded hand-off wait of any scan expired."""
        return scan_status(self.nv, c_void_p(self.streams[0].cuda_stream))

    def check_status(self):
        peer, scan = self.peer_status(), self.scan_status()
        assert peer == [0] * self.world, f"a bounded wait of the gradient exchange expired (peer_status per rank {peer})"
        assert scan == 0, "a bounded hand-off wait of a scan kernel expired (r2d2_scan_status)"

    def close(self):
        """Completes every pending finish and synchronises before any learner is destroyed or buffer freed (no rank may
        still read a peer's gradient block).  Returns (peer_status, scan_status) per rank."""
        if self.closed:
            return None
        self.flush()
        status = self.peer_status(), self.scan_status()
        for eng in self.engines:
            eng._pending_finish = False
            eng.close()
        self.engines, self.bufs, self.blocks = [], [], []
        self.closed = True
        return status

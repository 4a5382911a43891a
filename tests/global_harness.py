"""Global sampling in an in-process data-parallel group on one device (tests/peer_harness.py's PeerGroup): W engines with
PathConfig(global_sampling=True), each with its batch slots in a plain same-device buffer of the W-rank layout, each fed
by its own DeviceReplay shard attached to the group.

`global_schedule` is the call sequence of LearnerEngine.step / run_loop in peer mode with the global write-back and draw
in place of the prefetch hook (pipelined) or between the steps (sequential): the write-back's two stages, then - in the
hook, after the fill slot moved to the other slot (LearnerEngine._run_prefetch) - the draw's three stages.  `GlobalRun`
issues it group by group through DeviceReplay.global_write_back / global_draw (the code sample_into and
update_priorities run once attached), so every bounded wait finds its flags already raised."""
from __future__ import annotations

import numpy as np

from learner_harness import episode
from peer_harness import PeerGroup, peer_schedule

WRITE_BACK = [("write_back", 0), ("write_back", 1)]
DRAW = [("draw", 0), ("draw", 1), ("draw", 2)]


def global_schedule(steps: int, target_interval: int, prefetch: bool):
    """One list of calls per step: the first draw before step 0; pipelined, every prefetch hook becomes write-back +
    slot switch + draw; sequential, every step after the first is preceded by the previous batch's write-back and the
    draw into the same slot (run_loop's order)."""
    out = []
    for i, calls in enumerate(peer_schedule(steps, target_interval, prefetch)[:-1]):
        seq = list(DRAW) if i == 0 else ([] if prefetch else WRITE_BACK + DRAW)
        for c in calls:
            seq += WRITE_BACK + [("next_slot",)] + DRAW if c[0] == "prefetch" else [c]
        out.append(seq)
    return out


def make_shard(E, cfg, rng, n_eps, p_lo, cap):
    """(shard, the host episodes fed to it, oldest first)."""
    eps = [episode(rng, cfg, int(rng.integers(cfg.rows + 8, cfg.rows + 60)), p_lo=p_lo) for _ in range(n_eps)]
    rp = E.DeviceReplay(cfg, capacity_rows=cap)
    rp.add_episodes(eps)
    return rp, eps


class GlobalRun:
    def __init__(self, E, W, kw, seed=1, data_seed=3):
        import torch
        self.torch, self.E, self.W = torch, E, W
        self.g = PeerGroup(W, dict(kw, global_sampling=True), seed=seed)
        self.cfg = self.g.engines[0].cfg
        lay = self.g.engines[0].global_layout(W)
        self.bufs = [torch.zeros(int(lay.bytes) // 4, dtype=torch.float32, device="cuda") for _ in range(W)]
        ptrs = [b.data_ptr() for b in self.bufs]
        rng = np.random.default_rng(data_seed)
        self.shards, self.episodes = [], []     # per rank: its shard, the host episodes fed to it
        for r, eng in enumerate(self.g.engines):
            eng.use_global_slots(self.bufs[r], lay)
            eng.global_peer_ptrs, eng._rank = ptrs, r
            # unequal shards: sizes, masses (p_lo) and one small ring that wrapped and evicted
            cap = 600 if r == 1 else 6000
            rp, eps = make_shard(E, self.cfg, rng, 14 if r == 1 else 6 + 4 * r, 0.01 if r % 2 else 0.3, cap)
            rp.attach_group(eng)
            self.shards.append(rp)
            self.episodes.append(eps)
        torch.cuda.synchronize()
        self.gens = [torch.Generator(device="cuda").manual_seed(100 + r) for r in range(W)]
        self.draws = []          # per draw: (restated shard, leaf) and the device's

    def levels(self):
        return [[rp.tree_level(l).cpu().numpy() for l in range(rp.stats()["tree_levels"])] for rp in self.shards]

    def slot_cat(self, what, slot=None):
        """One slot's `what` of every rank, concatenated along the batch axis (rank order = global draw order)."""
        dim = {"obs": 1, "act": 1, "rew": 1, "term": 1, "states": 2}.get(what, 0)
        return self.torch.cat([e._slots[e._fill_slot if slot is None else slot][what] for e in self.g.engines], dim)

    def run(self, steps, prefetch, on_critic=None):
        from oracle import global_sumtree as gs
        g, torch = self.g, self.torch
        pending_u, lv = None, None
        for calls in global_schedule(steps, self.cfg.target_interval, prefetch):
            for c in calls:
                name = c[0]
                if name == "write_back":
                    g._issue(lambda r, eng, s, st=c[1]: self.shards[r].global_write_back(eng.leaf_idx, eng.priority, st))
                elif name == "next_slot":
                    g._issue(lambda r, eng, s: eng._bind_slot(1 - eng._fill_slot))
                elif name == "draw":
                    if c[1] == 0:
                        g.sync()
                        lv = self.levels()
                        pending_u = [torch.rand(self.cfg.batch, device="cuda", generator=gen) for gen in self.gens]
                        g.sync()                     # drawn on the default stream; the rank streams read them
                    g._issue(lambda r, eng, s, st=c[1]: self.shards[r].global_draw(eng, st, u=pending_u[r]))
                    if c[1] == 2:
                        g.sync()
                        ref = gs.global_draw(lv, torch.cat(pending_u).cpu().numpy())
                        got = (self.slot_cat("shard").cpu().numpy().astype(np.int64), self.slot_cat("leaf_idx").cpu().numpy())
                        self.draws.append((ref, got))
                else:
                    g._call(*c)
                    if name == "actor_phase":          # PeerGroup.flush completes the last deferred finish phase
                        g.pending = True
                    elif name == "finish_phase":
                        g.pending = None
                    if name == "critic_phase" and on_critic is not None:
                        g.sync()
                        on_critic(self.g.engines[0]._lib_slot)
        g.flush()

    def status(self):
        return [rp.global_status() for rp in self.shards]

    def close(self):
        out = self.g.close()
        for rp in self.shards:
            rp.close()
        return out


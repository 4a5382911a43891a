"""Global sampling over W replay shards on one GPU: W in-process ranks on same-device buffers, every stage issued for
all ranks before the next stage starts (one stream), so every bounded wait finds its flags already raised.

W = 1 is the local draw bit for bit; at W = 2, 3, 4, 8 (unequal shards, one without mass, one with nearly all of it,
one whose ring wrapped and evicted) every draw restates on the device trees (oracle/global_sumtree.py), every slot holds
the owning shard's rows, the weights are the global batch's, and after a write-back with a leaf drawn by two ranks every
tree level equals the C tree's."""
from ctypes import byref, c_int, c_void_p

import numpy as np
import pytest
import torch

from oracle import global_sumtree as gs
from oracle.sumtree import SumTreeOracle
from r2d2_b200 import engine as E
from r2d2_b200 import native as nv

pytestmark = pytest.mark.gpu

CFG = dict(obs=7, act=3, hidden=32, batch=16, burn_in=4, learning=6, n_step=2)


def _shard(cfg, rng, cap, n_eps, mass):
    rp = E.DeviceReplay(cfg, capacity_rows=cap)
    for _ in range(n_eps):
        n = int(rng.integers(cfg.rows + 4, cfg.rows + 40))
        ns = n - cfg.rows + 1
        pr = (rng.uniform(0.01, 1, ns) * mass).astype(np.float32)
        rp.add_episode(rng.standard_normal((n, cfg.obs)).astype(np.float32),
                       rng.uniform(-1, 1, (n, cfg.act)).astype(np.float32),
                       rng.standard_normal(n).astype(np.float32), (rng.random(n) < 0.05).astype(np.float32),
                       rng.standard_normal((ns, 4, 2, cfg.hidden)).astype(np.float32), pr)
    return rp


def _shards(cfg, W, rng):
    out = []
    for k in range(W):
        if k == 1 and W > 2:
            out.append(_shard(cfg, rng, 600, 3, 0.0))          # no mass: never chosen, still trains
        elif k == 2:
            out.append(_shard(cfg, rng, 4000, 20, 200.0))      # nearly all the mass
        elif k == 3:
            out.append(_shard(cfg, rng, 300, 40, 1.0))         # ring wrapped: rows evicted and reused
        else:
            out.append(_shard(cfg, rng, 2000 + 500 * k, 8, 0.3 + k))
    return out


class Group:
    def __init__(self, cfg, shards):
        self.cfg, self.shards, self.W = cfg, shards, len(shards)
        self.lib = nv.lib()
        self.lay = nv.GlobalLayout()
        nv.check(self.lib.r2d2_global_layout_for(cfg.rows, cfg.batch, cfg.obs, cfg.act, cfg.hidden, self.W,
                                                 byref(self.lay)))
        self.bufs = [torch.zeros(int(self.lay.bytes) // 4, dtype=torch.float32, device="cuda") for _ in shards]
        torch.cuda.synchronize()
        ptrs = (c_void_p * self.W)(*[b.data_ptr() for b in self.bufs])
        for r, rp in enumerate(shards):
            nv.check(self.lib.r2d2_replay_attach_group(rp._h, r, self.W, cfg.batch, ptrs, self.lay.bytes))
        self.stream = nv.current_stream()

    def view(self, rank, slot, what):
        c, lay = self.cfg, self.lay
        T, B = c.rows, c.batch
        shp = {"obs": ((T, B, c.obs), "<f4"), "act": ((T, B, c.act), "<f4"), "rew": ((T, B), "<f4"),
               "term": ((T, B), "<f4"), "states": ((4, 2, B, c.hidden), "<f4"), "leaf_idx": ((B,), "<i8"),
               "shard": ((B,), "<i4"), "is_weight": ((B,), "<f4"), "uniforms": ((B,), "<f4")}[what]
        p = self.bufs[rank].data_ptr() + int(lay.slot_offset[slot]) + int(getattr(lay, "off_" + what))
        return torch.as_tensor(nv._RawView(p, *shp), device="cuda")

    def draw(self, slot, us, weighted, beta):
        for r in range(self.W):
            self.view(r, slot, "uniforms").copy_(us[r])
        for stage in (0, 1, 2):
            for rp in self.shards:
                nv.check(self.lib.r2d2_replay_global_draw(rp._h, stage, slot, int(weighted), beta, self.stream))
        torch.cuda.synchronize()

    def write_back(self, slot, prios):
        for stage in (0, 1):
            for r, rp in enumerate(self.shards):
                nv.check(self.lib.r2d2_replay_global_write_back(rp._h, stage, nv.dptr(self.view(r, slot, "leaf_idx"), torch.int64),
                                                                nv.dptr(self.view(r, slot, "shard"), torch.int32),
                                                                nv.dptr(prios[r]), self.stream))
        torch.cuda.synchronize()

    def status(self):
        out = []
        for rp in self.shards:
            st = c_int(0)
            nv.check(self.lib.r2d2_replay_global_status(rp._h, byref(st), self.stream))
            out.append(st.value)
        return out


def _levels(rp):
    return [rp.tree_level(l).cpu().numpy() for l in range(rp.stats()["tree_levels"])]


def _host_gather(cfg, rp, leaf):
    T, B = cfg.rows, leaf.numel()
    out = {"obs": torch.zeros(T, B, cfg.obs, device="cuda"), "act": torch.zeros(T, B, cfg.act, device="cuda"),
           "rew": torch.zeros(T, B, device="cuda"), "term": torch.zeros(T, B, device="cuda"),
           "states": torch.zeros(4, 2, B, cfg.hidden, device="cuda")}
    nv.check(nv.lib().r2d2_replay_gather(rp._h, nv.dptr(leaf, torch.int64), B, *[nv.dptr(out[k]) for k in
                                                                                ("obs", "act", "rew", "term", "states")],
                                         nv.current_stream()))
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("weighted", [False, True])
def test_w1_is_the_local_draw(weighted):
    cfg = E.PathConfig(**CFG)
    rng = np.random.default_rng(11)
    rp = _shard(cfg, rng, 3000, 12, 1.0)
    local = _shard(cfg, np.random.default_rng(11), 3000, 12, 1.0)
    g = Group(cfg, [rp])
    eng = E.LearnerEngine(cfg, seed=1)
    eng.importance_weighting = weighted
    gen = torch.Generator(device="cuda").manual_seed(5)
    for it in range(3):
        u = torch.rand(cfg.batch, device="cuda", generator=gen)
        u[0] = 1.0 - 2.0 ** -24
        slot = it % 2
        g.draw(slot, [u], weighted, 0.6)
        local.sample_into(eng, u=u, beta=0.6)
        torch.cuda.synchronize()
        assert torch.equal(g.view(0, slot, "leaf_idx"), eng.leaf_idx)
        for k in ("obs", "act", "rew", "term", "states"):
            assert torch.equal(g.view(0, slot, k), getattr(eng, k)), k
        if weighted:
            assert torch.equal(g.view(0, slot, "is_weight"), eng.is_weight)
        prio = torch.rand(cfg.batch, device="cuda", generator=gen)
        g.write_back(slot, [prio])
        local.update_priorities(eng.leaf_idx, prio)
        torch.cuda.synchronize()
        for a, b in zip(_levels(rp), _levels(local)):
            assert np.array_equal(a, b)
    assert g.status() == [0]
    eng.close()


@pytest.mark.parametrize("W", [2, 3, 4, 8])
def test_global_draw_gather_weights_write_back(W):
    cfg = E.PathConfig(**CFG)
    rng = np.random.default_rng(100 + W)
    shards = _shards(cfg, W, rng)
    g = Group(cfg, shards)
    gen = torch.Generator(device="cuda").manual_seed(W)
    B = cfg.batch
    for it in range(3):
        slot = it % 2
        us = [torch.rand(B, device="cuda", generator=gen) for _ in range(W)]
        lv = [_levels(rp) for rp in shards]
        g.draw(slot, us, True, 0.6)
        shard, leaf, val = gs.global_draw(lv, torch.cat(us).cpu().numpy())
        got_leaf = torch.cat([g.view(c, slot, "leaf_idx") for c in range(W)]).cpu().numpy()
        got_shard = torch.cat([g.view(c, slot, "shard") for c in range(W)]).cpu().numpy()
        assert np.array_equal(got_shard, shard) and np.array_equal(got_leaf, leaf)
        if W > 2:
            assert not (shard == 1).any(), "the shard without mass was drawn"
        else:
            assert set(shard.tolist()) == {0, 1}, "W = 2: both shards hold mass and both are drawn from"
        w = torch.cat([g.view(c, slot, "is_weight") for c in range(W)]).cpu().numpy()
        ref_w = gs.is_weights(val, 0.6)
        np.testing.assert_allclose(w, ref_w, rtol=2e-6)
        assert w[np.argmin(np.where(val > 0, val, np.inf))] == 1.0
        for c in range(W):
            for k in set(shard[c * B:(c + 1) * B].tolist()):
                cols = np.nonzero(shard[c * B:(c + 1) * B] == k)[0]
                own = g.view(c, slot, "shard") == k          # other shards' leaves may lie past this shard's ring
                ref = _host_gather(cfg, shards[k], torch.where(own, g.view(c, slot, "leaf_idx"), 0))
                for name in ("obs", "act", "rew", "term"):
                    assert torch.equal(g.view(c, slot, name)[:, cols], ref[name][:, cols]), (c, k, name)
                assert torch.equal(g.view(c, slot, "states")[:, :, cols], ref["states"][:, :, cols]), (c, k)
        # write-back: rank W-1 trained the same row as rank 0's column 0; the higher global index must win
        g.view(W - 1, slot, "leaf_idx")[0] = g.view(0, slot, "leaf_idx")[0]
        g.view(W - 1, slot, "shard")[0] = g.view(0, slot, "shard")[0]
        prios = [torch.rand(B, device="cuda", generator=gen) for _ in range(W)]
        trees = []
        for k, rp in enumerate(shards):
            t = SumTreeOracle(rp.stats()["capacity_rows"])
            t.set_range(0, lv[k][0][:rp.stats()["capacity_rows"]])
            trees.append(t)
        rec_leaf = torch.cat([g.view(c, slot, "leaf_idx") for c in range(W)]).cpu().numpy()
        rec_shard = torch.cat([g.view(c, slot, "shard") for c in range(W)]).cpu().numpy()
        g.write_back(slot, prios)
        gs.write_back(trees, rec_leaf, rec_shard, torch.cat(prios).cpu().numpy())
        for k, rp in enumerate(shards):
            dev = _levels(rp)
            for l in range(trees[k].levels):
                assert np.array_equal(dev[l], trees[k].level(l)), (k, l)
    assert g.status() == [0] * W

"""Global sampling over W replay shards, restated on the C sum trees (oracle/global_sumtree.py): at W = 1 it is the
single tree's draw, and over many draws it samples the union of the shards in proportion to the stored leaves."""
import numpy as np
import pytest
from scipy import stats

from oracle import global_sumtree as gs
from oracle.sumtree import SumTreeOracle


def _tree(cap, rng, mass=1.0, sparse=0.5):
    t = SumTreeOracle(cap)
    v = rng.uniform(0.01, 1.0, cap).astype(np.float32) * np.float32(mass)
    v[rng.random(cap) < sparse] = 0
    t.set_range(0, v)
    return t, v


@pytest.mark.parametrize("cap", [31, 1000, 40000])
def test_w1_equals_single_tree(cap):
    rng = np.random.default_rng(cap)
    t, _ = _tree(cap, rng)
    u = rng.random(4096).astype(np.float32)
    u[:16] = np.float32(1.0) - np.float32(2.0 ** -24) * np.arange(1, 17, dtype=np.float32)   # residuals at the total
    shard, leaf, val = gs.global_draw([gs.levels_of(t)], u)
    assert (shard == 0).all()
    assert np.array_equal(leaf, t.sample(u))
    assert np.array_equal(val, t.level(0)[leaf])


def test_chi_square_against_global_proportions():
    rng = np.random.default_rng(7)
    caps, masses = [3000, 500, 2000, 1200], [1.0, 0.0, 40.0, 0.05]    # one empty shard, one holding nearly all mass
    trees, leaves = [], []
    for c, m in zip(caps, masses):
        t, v = _tree(c, rng, m, sparse=0.7)
        if m == 0.0:
            t.set_range(0, np.zeros(c, np.float32))
            v = np.zeros(c, np.float32)
        trees.append(t)
        leaves.append(v)
    n = 1 << 20
    u = rng.random(n).astype(np.float32)
    shard, leaf, _ = gs.global_draw([gs.levels_of(t) for t in trees], u)
    flat = np.concatenate(leaves).astype(np.float64)
    offs = np.cumsum([0] + caps[:-1])
    counts = np.bincount(offs[shard] + leaf, minlength=flat.size)
    assert counts[flat == 0].sum() == 0, "a zero leaf was drawn"
    p = flat / flat.sum()
    # pool the leaves into bins of >= 50 expected draws, then a chi-square test at 1e-3
    order = np.argsort(p)
    exp, obs, acc_e, acc_o = [], [], 0.0, 0
    for i in order[p[order] > 0]:
        acc_e += n * p[i]
        acc_o += counts[i]
        if acc_e >= 50:
            exp.append(acc_e); obs.append(acc_o); acc_e, acc_o = 0.0, 0
    if acc_e > 0:
        exp[-1] += acc_e; obs[-1] += acc_o
    exp, obs = np.asarray(exp), np.asarray(obs)
    pv = stats.chisquare(obs, exp * obs.sum() / exp.sum()).pvalue
    assert pv > 1e-3, pv
    per_shard = np.bincount(shard, minlength=4) / n
    assert per_shard[1] == 0.0
    assert per_shard[2] > 0.9, per_shard            # far from 1/W: the shard with the mass supplies the batch
    mass = np.asarray([v.astype(np.float64).sum() for v in leaves])
    assert np.allclose(per_shard, mass / mass.sum(), atol=3e-3)


def test_write_back_filters_by_shard_and_last_global_index_wins():
    rng = np.random.default_rng(3)
    trees = [_tree(200, rng)[0] for _ in range(3)]
    ref = [_tree(200, np.random.default_rng(3))[0] for _ in range(3)]
    for t, r in zip(trees, ref):
        r.set_range(0, t.level(0))
    leaf = np.array([5, 5, 7, 5, 9, 7], np.int64)
    shard = np.array([0, 1, 0, 0, 2, 0], np.int64)
    prio = np.array([1, 2, 3, 4, 5, 6], np.float32)
    gs.write_back(trees, leaf, shard, prio)
    assert trees[0].level(0)[5] == 4 and trees[0].level(0)[7] == 6
    assert trees[1].level(0)[5] == 2 and trees[2].level(0)[9] == 5
    for t in trees:
        lv = t.level(0)
        for l in range(1, t.levels):
            lv = lv.reshape(-1, 32) if lv.size % 32 == 0 else np.pad(lv, (0, -lv.size % 32)).reshape(-1, 32)
            s = np.zeros(lv.shape[0], np.float32)
            for k in range(32):
                s = (s + lv[:, k]).astype(np.float32)
            assert np.array_equal(s[:t.level(l).size], t.level(l))
            lv = t.level(l)

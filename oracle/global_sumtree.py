"""Restatement of global sampling over W replay shards (csrc/replay.cu global_draw_kernel, tree_update_kernel with a
shard filter) on the C sum trees of oracle/sumtree_oracle.c (TEST INFRASTRUCTURE).

The W shard roots are one more tree level above the shards, in rank order.  Global draw j: r = u_j * total, total the
left-to-right fp32 sum of the roots; the roots are walked as a node's 32 children are (first root with r < root, else
r -= root); if rounding pushes r past the last root, the last non-empty shard is taken with the residual as it stood
before that shard; then the owning shard's tree is descended with the residual by the C tree's rule.  Every operation is
one fp32 operation (numpy float32), so the result is the device's bit for bit.
"""
from __future__ import annotations

import numpy as np

from .sumtree import SumTreeOracle

F = np.float32
K = 32


def descend(levels, r):
    """Leaf index and leaf value for residuals r (float32 array) in the tree `levels` (level 0 = leaves, last = root):
    st_sample's descent, vectorised, starting from a given residual."""
    r = np.array(r, dtype=F, copy=True)
    n = r.size
    idx = np.zeros(n, np.int64)
    val = np.zeros(n, F)
    for lvl in range(len(levels) - 1, 0, -1):
        child = levels[lvl - 1]
        c = np.zeros((n, K), F)
        base = idx * K
        for k in range(K):
            pos = base + k
            ok = pos < child.size
            c[ok, k] = child[pos[ok]]
        pick = np.full(n, -1, np.int64)
        for k in range(K):
            open_ = pick < 0
            hit = open_ & (r < c[:, k])
            pick[hit] = k
            val[hit] = c[hit, k]
            miss = open_ & ~hit
            r[miss] = (r[miss] - c[miss, k]).astype(F)
        fb = pick < 0
        if fb.any():
            nz = c[fb] > 0
            last = np.where(nz.any(axis=1), K - 1 - np.argmax(nz[:, ::-1], axis=1), 0)
            cl = c[fb][np.arange(fb.sum()), last] * nz.any(axis=1)
            pick[fb] = last
            r[fb] = (cl.astype(F) * F(0.99999994)).astype(F)
            val[fb] = cl.astype(F)
        idx = idx * K + pick
    return idx, val


def pick_shards(roots, u):
    """(shard, residual) of global draws with uniforms u over shard roots `roots` (float32 [W])."""
    roots = np.asarray(roots, F)
    u = np.asarray(u, F)
    total = F(0)
    for x in roots:
        total = F(total + x)
    r0 = (u * total).astype(F)
    r = r0.copy()
    pick = np.full(u.size, -1, np.int64)
    for k, x in enumerate(roots):
        open_ = pick < 0
        hit = open_ & (r < x)
        pick[hit] = k
        miss = open_ & ~hit
        r[miss] = (r[miss] - x).astype(F)
    fb = pick < 0
    if fb.any():
        nz = np.nonzero(roots > 0)[0]
        p = int(nz[-1]) if nz.size else 0
        pick[fb] = p
        rr = r0[fb].copy()
        for k in range(p):
            rr = (rr - roots[k]).astype(F)
        r[fb] = rr
    return pick, r


def global_draw(shard_levels, u):
    """shard_levels[k] = level arrays of shard k's tree.  Returns (shard, leaf, leaf value) per global draw."""
    roots = [lv[-1][0] for lv in shard_levels]
    shard, r = pick_shards(roots, u)
    leaf = np.zeros(shard.size, np.int64)
    val = np.zeros(shard.size, F)
    for k, lv in enumerate(shard_levels):
        m = shard == k
        if m.any():
            leaf[m], val[m] = descend(lv, r[m])
    return shard, leaf, val


def is_weights(leaf_val, beta):
    """is_weight_kernel over one (global) batch of drawn leaf values, in float32 except powf (left to the caller's
    tolerance: the device's powf is not restated)."""
    v = np.asarray(leaf_val, F)
    pos = v > 0
    m = v[pos].min() if pos.any() else F(np.inf)
    out = np.ones_like(v)
    if beta != 0:
        out[pos] = np.power((m / v[pos]).astype(F).astype(np.float64), beta).astype(F)
    return out


def write_back(trees, leaf, shard, prio):
    """Apply W*B records in global-index order: each shard takes the records that land in it (the last of a duplicate
    leaf wins, as st_update_batch's in-order writes do).  trees: SumTreeOracle per shard; prio already as stored."""
    leaf, shard, prio = np.asarray(leaf, np.int64), np.asarray(shard, np.int64), np.asarray(prio, F)
    for k, t in enumerate(trees):
        m = shard == k
        if m.any():
            t.update_batch(leaf[m], prio[m])


def levels_of(tree: SumTreeOracle):
    return [tree.level(l) for l in range(tree.levels)]

"""The data-parallel gradient exchange (csrc/peer.cu: signal / slice sum / wait, placed inside the learner's phases) on
one GPU: W in-process ranks on same-device buffers (tests/peer_harness.py), issued group by group in the order
LearnerEngine.step uses in the "peer" mode.

 (a) exchange bits: every rank's sums are numpy's float32 0 + g_0 + ... + g_{W-1} over the ranks' gradient blocks, the
     same bits on every rank, the pad tail zero; W up to 16 (the second 8-peer chunk, padding for W not a power of two)
     and cfg-3 widths (a slice larger than one grid pass), four iterations so that flags and the CTA ticket are reused;
 (b) W = 2 on identical shards is one engine on that shard bit for bit (fl(0 + g + g) * 1/2 = g), with every optimiser
     and TD option and the pipelined step;
 (c) W = 2, 3, 4 on disjoint shards of one global batch against the float64 oracle of the global batch;
 (d) attach_peers' argument checks and the six exchange launches per iteration."""
import numpy as np
import pytest
import torch

from conftest import rel_l2
from learner_harness import oracle_for
from oracle import learner_oracle as lo
from oracle import ref_port
from peer_harness import PeerGroup, split_batch

pytestmark = pytest.mark.gpu

ERR_ARG = -2
SMALL = dict(obs=6, act=2, hidden=64, batch=8, burn_in=4, learning=6, n_step=2)
ITERS = 6
# optimiser / TD options of (b) and (c): PathConfig fields, and whether the batch carries importance weights
OPTIONS = {
    "defaults": ({}, False),
    "clip_polyak_every": (dict(grad_clip_norm=0.05, target_tau=0.05, target_interval=1), False),
    "polyak_every_3": (dict(target_tau=0.3, target_interval=3), False),
    "is_weights": (dict(is_exponent=0.6), True),
    "invertible_abs": (dict(value_rescaling="invertible", rescaling_eps=1e-3, priority_metric="abs"), False),
}


@pytest.fixture(scope="module")
def E():
    from r2d2_b200 import engine
    engine.nv.lib()
    return engine


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def global_batches(kw, n, seed, weights):
    pc = ref_port.PathConfig(**kw)
    rng = np.random.default_rng(seed + 1000)
    out = []
    for i in range(n):
        b = ref_port.synthetic_batch(pc, seed=seed + i)
        if weights:
            b["is_weight"] = rng.uniform(0.05, 1.0, kw["batch"]).astype(np.float32)
        out.append(b)
    return out


def state(eng):
    out = {f"flat.{n}": eng.flat[n].cpu().numpy() for n in ("actor", "critic", "target_actor", "target_critic")}
    for d, name in ((eng.exp_avg, "m"), (eng.exp_avg_sq, "v")):
        out.update({f"{name}.{n}": d[n].cpu().numpy() for n in ("actor", "critic")})
    return out


def assert_same_state(a, b, what):
    assert a.keys() == b.keys()
    for k in a:
        assert np.array_equal(u32(a[k]), u32(b[k])), f"{what}: {k} differs"


# ------------------------------------------------------------------------------------------------ (a) exchange bits
def _check_exchange(g, net, it, seen):
    W = g.world
    grads = [g.block("grads", net, r, pad=True) for r in range(W)]
    sums = [g.block("sums", net, r, pad=True) for r in range(W)]
    n = g.n[net]
    want = np.zeros_like(grads[0])
    for x in grads:                                   # rank order, float32, left to right
        want = want + x
    for r in range(W):
        assert np.array_equal(u32(sums[r]), u32(want)), \
            f"{net} it {it}: rank {r}'s sums are not 0 + g_0 + ... + g_{W - 1} (first bad index " \
            f"{int(np.flatnonzero(u32(sums[r]) != u32(want))[0])} of {n})"
        assert not grads[r][n:].any() and not sums[r][n:].any(), f"{net} it {it}: pad tail of rank {r} is not zero"
    assert all(np.count_nonzero(x[:n]) > n // 2 for x in grads), f"{net} it {it}: gradient blocks mostly zero"
    if W > 1:
        assert not np.array_equal(grads[0], grads[1]), f"{net} it {it}: ranks trained on the same data"
    seen.add((net, it))


EXCHANGE = [(W, H) for W in (2, 3, 5, 8, 9, 16) for H in (32, 64)]


@pytest.mark.parametrize("W,H", EXCHANGE, ids=[f"W{w}-H{h}" for w, h in EXCHANGE])
def test_exchange_sums_are_rank_ordered_float32_sums(E, W, H):
    per_rank = 16 // W                                # W = 16: one sequence per rank
    kw = dict(obs=5, act=3, hidden=H, batch=per_rank * W, burn_in=3, learning=5, n_step=2)
    _exchange_run(E, W, kw, per_rank, iters=4)


@pytest.mark.parametrize("W", [2, 3])
def test_exchange_sums_at_cfg3_widths(E, W):
    kw = dict(obs=376, act=17, hidden=512, batch=4 * W, burn_in=2, learning=4, n_step=2)
    g = _exchange_run(E, W, kw, 4, iters=4)
    assert g["slice_vec"] > 132 * 512, g               # one rank's slice takes more than one pass of the grid


def _exchange_run(E, W, kw, per_rank, iters):
    g = PeerGroup(W, dict(kw, batch=per_rank))
    try:
        shards = [split_batch(b, W) for b in global_batches(kw, iters, seed=11 * W + kw["hidden"], weights=False)]
        seen = set()
        g.run(shards, on_iteration=lambda it: _check_exchange(g, "critic", it, seen),
              on_finish=lambda it: _check_exchange(g, "actor", it, seen))
        assert seen == {(net, it) for net in ("critic", "actor") for it in range(iters)}
        g.check_status()
        info = {"slice_vec": g.padded["critic"] // 4 // W, "n_critic": g.n["critic"]}
    finally:
        g.close()
    return info


# ------------------------------------------------------------------------------------------------ (b) bit identity
def _single_run(E, cfg_kw, batches, prefetch):
    """One engine on the batches (plain loop, or the pipelined step drawing the next batch from its hook): per iteration
    q, target, priority, losses, grad_norms, then the final state."""
    eng = E.LearnerEngine(E.PathConfig(**cfg_kw), seed=1)
    per_it = []

    def record():
        torch.cuda.synchronize()
        per_it.append({k: getattr(eng, k).cpu().numpy() for k in ("q_value", "target_q_value", "priority", "losses",
                                                                   "grad_norms")})
    eng.set_batch(batches[0])
    for it in range(ITERS):
        if prefetch:
            eng.step(prefetch=lambda e, used, it=it: e.set_batch(batches[it + 1]))
        else:
            if it:
                eng.set_batch(batches[it])
            eng.step()
        record()
    out = state(eng)
    eng.close()
    return per_it, out


def _group_records(g):
    """Callbacks for PeerGroup.run that record, per rank and iteration, what _single_run records."""
    rec = [[{} for _ in range(ITERS)] for _ in range(g.world)]

    def on_iteration(it):
        for r, eng in enumerate(g.engines):
            rec[r][it].update({k: getattr(eng, k).cpu().numpy() for k in ("q_value", "target_q_value", "priority",
                                                                           "losses")})
            rec[r][it]["critic_norm"] = eng.grad_norms[0].item()

    def on_finish(it):
        for r, eng in enumerate(g.engines):
            rec[r][it]["actor_norm"] = eng.grad_norms[1].item()
            rec[r][it]["state"] = state(eng)
    return rec, on_iteration, on_finish


MATRIX = [(o, p) for o in OPTIONS for p in (False, True)]
MATRIX_IDS = [f"{o}-{'pipelined' if p else 'plain'}" for o, p in MATRIX]


@pytest.mark.parametrize("option,prefetch", MATRIX, ids=MATRIX_IDS)
def test_two_ranks_on_identical_shards_are_one_engine_bit_for_bit(E, option, prefetch):
    extra, weights = OPTIONS[option]
    kw = dict(SMALL, **extra)
    batches = global_batches(SMALL, ITERS + 1, seed=70, weights=weights)
    single, single_state = _single_run(E, kw, batches, prefetch)
    g = PeerGroup(2, kw)
    try:
        rec, on_iteration, on_finish = _group_records(g)
        g.run([[b, b] for b in (batches if prefetch else batches[:ITERS])], prefetch=prefetch,
              on_iteration=on_iteration, on_finish=on_finish)
        g.check_status()
        for it in range(ITERS):
            for r in range(2):
                got = rec[r][it]
                want = single[it]
                for k in ("q_value", "target_q_value", "priority", "losses"):
                    assert np.array_equal(u32(got[k]), u32(want[k])), f"it {it} rank {r}: {k}"
                norms = np.asarray([got["critic_norm"], got["actor_norm"]], np.float32)
                assert np.array_equal(u32(norms), u32(want["grad_norms"])), f"it {it} rank {r}: grad_norms"
        for r in range(2):
            assert_same_state(rec[r][ITERS - 1]["state"], single_state, f"rank {r} final state")
    finally:
        g.close()


# ------------------------------------------------------------------------------------------------ (c) float64 parity
GLOBAL = dict(SMALL, batch=12)
_ORACLE = {}


def _oracle(E, option):
    """The float64 learner on the global batches, once per option set."""
    if option in _ORACLE:
        return _ORACLE[option]
    extra, weights = OPTIONS[option]
    cfg = E.PathConfig(**GLOBAL, **extra)
    gen = torch.Generator().manual_seed(1)                        # LearnerEngine(seed=1)'s initial nets
    actor = {k: v.numpy() for k, v in E.init_reference_params(cfg, False, gen).items()}
    critic = {k: v.numpy() for k, v in E.init_reference_params(cfg, True, gen).items()}
    batches = global_batches(GLOBAL, ITERS + 1, seed=90, weights=weights)
    ol = oracle_for(cfg, actor, critic)
    flat = lambda g: np.concatenate([np.asarray(g[k], np.float64).ravel() for k in lo.PARAM_KEYS])  # noqa: E731
    per_it = []
    for it in range(ITERS):
        ref = ol.iteration(batches[it])
        per_it.append(dict(q_value=ref["q_value"], target_q_value=ref["target_q_value"], td_sq=ref["average_td_loss"],
                           losses=(ref["critic_loss"], ref["actor_loss"]),
                           critic_grad=flat(ref["pre_clip_grad"]["critic"]), actor_grad=flat(ref["pre_clip_grad"]["actor"]),
                           norms=(ol.norms["critic"], ol.norms["actor"])))
    final = {}
    for net in ("actor", "critic"):
        final["flat." + net] = getattr(ol, net)
        final["flat.target_" + net] = getattr(ol, "target_" + net)
        final["m." + net] = {k: getattr(ol, net + "_adam")["m/" + k] for k in lo.PARAM_KEYS}
        final["v." + net] = {k: getattr(ol, net + "_adam")["v/" + k] for k in lo.PARAM_KEYS}
    _ORACLE[option] = (batches, per_it, final, cfg)
    return _ORACLE[option]


def _shard_priorities(td_sq, B, W, r, metric, eta=0.9):
    """learner.py:137's [b:-1:B] series over one rank's columns of the global td_sq [L, B]."""
    b = B // W
    flat = td_sq.reshape(-1, B)[:, r * b:(r + 1) * b].reshape(-1)
    flat = np.sqrt(flat) if metric == "abs" else flat
    return np.asarray([eta * flat[j:-1:b].max() + (1 - eta) * flat[j:-1:b].mean() for j in range(b)])


def _concat_shards(xs, L, A):
    return np.concatenate([x.reshape(L, -1, A) for x in xs], 1).reshape(-1, A)


PARITY = [(W, o, p) for W in (2, 3, 4) for o in OPTIONS for p in (False, True)]


@pytest.mark.parametrize("W,option,prefetch", PARITY,
                         ids=[f"W{w}-{o}-{'pipelined' if p else 'plain'}" for w, o, p in PARITY])
def test_disjoint_shards_against_float64(E, W, option, prefetch):
    batches, ref, final, cfg = _oracle(E, option)
    L, A, B = cfg.learning, cfg.act, cfg.batch
    extra, _ = OPTIONS[option]
    g = PeerGroup(W, dict(GLOBAL, batch=B // W, **extra))
    errs = {}
    clip = cfg.grad_clip_norm > 0

    def err(group, v):
        errs[group] = max(errs.get(group, 0.0), v)

    def replicas(it):
        s0 = state(g.engines[0])
        for r in range(1, W):
            assert_same_state(state(g.engines[r]), s0, f"it {it} rank {r} vs rank 0")

    def on_iteration(it):
        o = ref[it]
        engs = g.engines
        err("q", rel_l2(_concat_shards([e.q_value.cpu().numpy() for e in engs], L, A), o["q_value"]))
        err("target_q", rel_l2(_concat_shards([e.target_q_value.cpu().numpy() for e in engs], L, A), o["target_q_value"]))
        for r, e in enumerate(engs):
            want = _shard_priorities(o["td_sq"], B, W, r, cfg.priority_metric)
            err("priority", rel_l2(e.priority.cpu().numpy(), want))
        err("critic_loss", abs(np.mean([e.losses[0].item() for e in engs]) / o["losses"][0] - 1))
        err("actor_loss", abs(np.mean([e.losses[1].item() for e in engs]) / o["losses"][1] - 1))
        _sums_vs_oracle(0, it)

    def _sums_vs_oracle(net_i, it):
        net = ("critic", "actor")[net_i]
        sums = g.block("sums", net, 0).astype(np.float64)
        err(f"{net}_sums", rel_l2(sums / W, ref[it][net + "_grad"]))
        if clip:
            mine = [e.grad_norms[net_i].item() for e in g.engines]
            assert len(set(mine)) == 1, f"{net} norms differ between ranks: {mine}"
            err(f"{net}_norm_vs_sums", abs(mine[0] / (np.linalg.norm(sums) / W) - 1))
            err(f"{net}_norm_vs_oracle", abs(mine[0] / ref[it]["norms"][net_i] - 1))

    def on_finish(it):
        _sums_vs_oracle(1, it)
        replicas(it)

    try:
        g.run([split_batch(b, W) for b in (batches if prefetch else batches[:ITERS])], prefetch=prefetch,
              on_iteration=on_iteration, on_finish=on_finish)
        g.check_status()
        for name, mine in state(g.engines[0]).items():
            net = name.split(".", 1)[1]
            theirs = final[name]
            views = E.flat_views(torch.as_tensor(mine), cfg, "critic" in net)
            for k in lo.PARAM_KEYS:
                err(name.split(".")[0] + ("_target" if "target" in net else ""), rel_l2(views[k].numpy(), theirs[k]))
    finally:
        g.close()
    bounds = {"critic_sums": 1e-4, "actor_sums": 1e-4, "critic_norm_vs_sums": 1e-6, "actor_norm_vs_sums": 1e-6,
              "critic_norm_vs_oracle": 1e-4, "actor_norm_vs_oracle": 1e-4}
    print(f"\nDP parity W={W} {option} {'pipelined' if prefetch else 'plain'}: "
          + " ".join(f"{k}={v:.2e}" for k, v in sorted(errs.items())))
    bad = {k: v for k, v in errs.items() if not v < bounds.get(k, 1e-3)}
    assert not bad, bad


# ------------------------------------------------------------------------------------------------ (d) API edges
def test_attach_rejects_bad_arguments_and_the_learner_still_steps(E):
    from ctypes import c_void_p
    cfg = E.PathConfig(**SMALL)
    batch = ref_port.synthetic_batch(ref_port.PathConfig(**SMALL), seed=5)
    eng = E.LearnerEngine(cfg, seed=1)
    lay = E.nv.PeerLayout()
    E.nv.check(eng.lib.r2d2_learner_peer_layout(eng._h, 2, E.nv.byref(lay)))
    bufs = [torch.zeros(int(lay.bytes) // 4, device=eng.device) for _ in range(17)]
    ptrs = (c_void_p * 17)(*[b.data_ptr() for b in bufs])
    lib = eng.lib
    for rank, world in ((0, 1), (0, 17), (-1, 2), (2, 2), (5, 3)):
        assert lib.r2d2_learner_attach_peers(eng._h, rank, world, ptrs) == ERR_ARG, (rank, world)
    holed = (c_void_p * 3)(bufs[0].data_ptr(), None, bufs[2].data_ptr())
    assert lib.r2d2_learner_attach_peers(eng._h, 0, 3, holed) == ERR_ARG
    assert lib.r2d2_learner_attach_peers(None, 0, 2, ptrs) == ERR_ARG
    plain = E.LearnerEngine(cfg, seed=1)
    for e in (eng, plain):
        e.set_batch(batch)
        e.step()
        e.step()
    torch.cuda.synchronize()
    assert_same_state(state(eng), state(plain), "after refused attaches")
    assert not any(b.any() for b in bufs), "a refused attach wrote into a peer buffer"
    eng.close()
    plain.close()


def test_second_attach_is_refused(E):
    g = PeerGroup(2, SMALL)
    try:
        from ctypes import c_void_p
        ptrs = (c_void_p * 2)(*[b.data_ptr() for b in g.bufs])
        for r, eng in enumerate(g.engines):
            assert g.lib.r2d2_learner_attach_peers(eng._h, r, 2, ptrs) == ERR_ARG
        batches = global_batches(dict(SMALL, batch=16), 2, seed=3, weights=False)
        g.run([split_batch(b, 2) for b in batches])
        g.check_status()
    finally:
        g.close()


@pytest.mark.parametrize("option", ["defaults", "clip_polyak_every"])
def test_exchange_adds_six_launches_per_iteration(E, option):
    extra, _ = OPTIONS[option]
    kw = dict(SMALL, **extra)
    batches = global_batches(dict(SMALL, batch=16), 3, seed=4, weights=False)
    plain = E.LearnerEngine(E.PathConfig(**kw), seed=1)
    E.nv.check(plain.lib.r2d2_learner_set_overlap_actor_inputs(plain._h, 0))
    for b in batches:
        plain.set_batch(split_batch(b, 2)[0])
        plain.step()
    torch.cuda.synchronize()
    g = PeerGroup(2, kw)
    try:
        g.run([split_batch(b, 2) for b in batches], final_flush=False)    # the deferred finish of iteration 2 is due
        got = [e.launches_per_iteration for e in g.engines]
        g.flush()
        g.check_status()
    finally:
        g.close()
    assert got == [plain.launches_per_iteration + 6] * 2, (got, plain.launches_per_iteration)
    plain.close()

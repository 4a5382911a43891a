"""Prioritized replay on the GPU: the priority exponent alpha on the sum-tree leaves, the importance-sampling weights
of the weighted draw, the weighted critic loss of the learner, and that the defaults (alpha = 1, beta = 0) are the
unweighted library bit for bit."""
import numpy as np
import pytest
import torch

from conftest import rel_l2
from learner_harness import (REPLAY, SMALL, TOL, assert_two_gpu_replicas_stay_identical, episode, golden_case, oracle_for,
                             port_case, replay_fed_run, trained_dropin_learner)
from oracle import learner_oracle as lo
from oracle.replay_model import ReplayModel
from oracle.sumtree import SumTreeOracle

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng_mod():
    from r2d2_b200 import engine
    return engine


def ingest(rp, model, eps):
    """One actor file into the shard and into its host model: the same rows, evictions and counter."""
    got = rp.add_episodes(eps)
    assert got == model.add_episodes(eps)
    return got[1]


def ingest_wrap_writeback(eng_mod, rp, cfg, cap, seed):
    """Three actor files into a small ring (the third wraps and evicts), then a write-back with duplicate leaves."""
    rng = np.random.default_rng(seed)
    model = ReplayModel.for_config(cfg, cap)
    evicted = 0
    for n_eps in (10, 10, 12):
        evicted += ingest(rp, model, [episode(rng, cfg, int(rng.integers(60, 160))) for _ in range(n_eps)])
    live = model.live_starts()
    leaf = np.concatenate([rng.choice(live, 200), rng.choice(live, 40)])
    leaf[-20:] = leaf[:20]                              # duplicates inside one write-back
    prio = rng.uniform(0.05, 3.0, leaf.size).astype(np.float32)
    rp.update_priorities(torch.as_tensor(leaf).cuda(), torch.as_tensor(prio).cuda())
    model.update_priorities(leaf, prio)
    return model, evicted


def tree_levels(rp):
    return [rp.tree_level(l).cpu().numpy().copy() for l in range(rp.stats()["tree_levels"])]


# ---------------------------------------------------------------------------------------------------- 1. defaults
def test_default_exponent_is_the_unexponentiated_tree(eng_mod):
    cfg = eng_mod.PathConfig(obs=4, act=2, hidden=8, batch=8, burn_in=4, learning=6, n_step=2)
    cap = 3000
    a = eng_mod.DeviceReplay(cfg, capacity_rows=cap)
    b = eng_mod.DeviceReplay(cfg, capacity_rows=cap)
    assert b.lib.r2d2_replay_set_priority_exponent(b._h, 1.0) == 0
    _, ev_a = ingest_wrap_writeback(eng_mod, a, cfg, cap, seed=1)
    _, ev_b = ingest_wrap_writeback(eng_mod, b, cfg, cap, seed=1)
    assert ev_a == ev_b > 0
    for la, lb in zip(tree_levels(a), tree_levels(b)):
        assert np.array_equal(la.view(np.uint32), lb.view(np.uint32))


@pytest.mark.parametrize("hidden,batch", [(256, 64), (512, 32)])
def test_weighting_at_beta_zero_is_the_unweighted_run(eng_mod, hidden, batch):
    runs = []
    for weighted in (False, True):
        def setup(eng, weighted=weighted):
            assert eng.importance_weighting == weighted
        runs.append(replay_fed_run(eng_mod, 6, setup=setup, beta=0.0, hidden=hidden, batch=batch,
                                   replay_cfg=eng_mod.PathConfig(**dict(REPLAY, hidden=hidden, batch=batch)),
                                   keep=("td_sq", "leaf_idx", "is_weight"), is_exponent=0.6 if weighted else 0.0))
    off, on = runs
    assert torch.equal(on["is_weight"], torch.ones_like(on["is_weight"]))
    for k in ("launches", "q_value", "target_q_value", "td_sq", "priority", "losses", "leaf_idx", "flat.actor",
              "flat.critic", "flat.target_actor", "flat.target_critic"):
        assert torch.equal(off[k], on[k]), k


# ---------------------------------------------------------------------------------------------------- 2. alpha
@pytest.mark.parametrize("alpha", [0.0, 0.6, 0.9])
def test_leaves_hold_priority_to_the_alpha(eng_mod, alpha):
    cfg = eng_mod.PathConfig(obs=4, act=2, hidden=8, batch=8, burn_in=4, learning=6, n_step=2,
                             priority_exponent=alpha)
    cap = 3000
    rp = eng_mod.DeviceReplay(cfg, capacity_rows=cap)
    model, evicted = ingest_wrap_writeback(eng_mod, rp, cfg, cap, seed=int(alpha * 10) + 3)
    assert evicted > 0
    leaves = rp.tree_level(0).cpu().numpy()[:cap]
    live = model.raw > 0
    want = model.raw[live].astype(np.float64) ** alpha
    assert np.abs(leaves[live] / want - 1.0).max() < 1e-6
    assert (leaves[~live] == 0).all()
    oracle = SumTreeOracle(cap)
    oracle.set_range(0, leaves)
    for l, lv in enumerate(tree_levels(rp)):
        assert np.array_equal(lv[:len(oracle.level(l))], oracle.level(l)), f"level {l}"
    # alpha is fixed once the shard holds data; out-of-range values are refused on an empty shard too
    assert rp.lib.r2d2_replay_set_priority_exponent(rp._h, 0.5) == -4          # R2D2_ERR_STATE
    empty = eng_mod.DeviceReplay(cfg, capacity_rows=256)
    for bad in (-0.1, 1.5, float("nan")):
        assert empty.lib.r2d2_replay_set_priority_exponent(empty._h, bad) == -2   # R2D2_ERR_ARG
    assert empty.lib.r2d2_replay_set_priority_exponent(empty._h, 0.3) == 0


# ---------------------------------------------------------------------------------------------------- 3. draw law
@pytest.mark.parametrize("alpha", [0.0, 0.6])
def test_draws_follow_priority_to_the_alpha(eng_mod, alpha):
    cfg = eng_mod.PathConfig(obs=3, act=1, hidden=4, batch=32, burn_in=4, learning=6, n_step=2,
                             priority_exponent=alpha)
    rng = np.random.default_rng(21)
    rp = eng_mod.DeviceReplay(cfg, capacity_rows=40000)
    model = ReplayModel.for_config(cfg, 40000)
    ingest(rp, model, [episode(rng, cfg, int(rng.integers(40, 120)), p_lo=2e-3) for _ in range(60)])
    starts = model.live_starts()
    n = 1 << 20
    u = torch.rand(n, device="cuda", generator=torch.Generator(device="cuda").manual_seed(4))
    cnt = np.bincount(rp.sample_indices(u).cpu().numpy(), minlength=40000)
    assert cnt.sum() == cnt[starts].sum()                                       # only valid starts are drawn
    p = model.raw[starts].astype(np.float64) ** alpha
    exp = p / p.sum() * n
    chi2 = ((cnt[starts] - exp) ** 2 / exp).sum() / len(starts)
    assert 0.85 < chi2 < 1.15, chi2
    if alpha == 0.0:
        assert np.allclose(exp, n / len(starts))


# ---------------------------------------------------------------------------------------------------- 4. weights
def test_importance_weights(eng_mod):
    kw = dict(obs=4, act=2, hidden=32, batch=256, burn_in=4, learning=6, n_step=2)
    rp = eng_mod.DeviceReplay(eng_mod.PathConfig(**kw, priority_exponent=0.9), capacity_rows=20000)
    rng = np.random.default_rng(8)
    rp.add_episodes([episode(rng, eng_mod.PathConfig(**kw), int(rng.integers(40, 200))) for _ in range(40)])
    eng = eng_mod.LearnerEngine(eng_mod.PathConfig(**kw, is_exponent=0.6))
    u = torch.rand(256, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    u[200:] = u[:56]                                                           # duplicate draws
    leaves = rp.tree_level(0).cpu().numpy()
    for beta in (0.6, 1.0, 0.25):
        rp.sample_into(eng, u=u, beta=beta)
        torch.cuda.synchronize()
        li, w = eng.leaf_idx.cpu().numpy(), eng.is_weight.cpu().numpy()
        lv = leaves[li].astype(np.float64)
        assert (lv > 0).all()
        want = (lv.min() / lv) ** beta
        assert np.abs(w / want - 1.0).max() < 1e-6, beta
        assert w.max() == np.float32(1.0) and (w > 0).all()
        assert np.array_equal(w[200:], w[:56])
        for l in np.unique(li):
            assert np.unique(w[li == l]).size == 1
    rp.sample_into(eng, u=u)                                                   # default: cfg.is_exponent
    torch.cuda.synchronize()
    assert np.abs(eng.is_weight.cpu().numpy() / ((lv.min() / lv) ** 0.6) - 1.0).max() < 1e-6
    rp.sample_into(eng, u=u, beta=0.0)
    torch.cuda.synchronize()
    assert (eng.is_weight.cpu().numpy() == 1.0).all()
    with pytest.raises(ValueError):
        rp.sample_into(eng, u=u, beta=1.5)


# ---------------------------------------------------------------------------------------------------- 5. learner parity
def _check_weighted_iteration(eng_mod, cfg, actor, critic, batch, w):
    """One weighted iteration against the float64 oracle; td_sq / priorities bit-identical to the unweighted engine."""
    eng = eng_mod.LearnerEngine(cfg)
    eng.load_state_dicts(actor, critic)
    eng.set_batch(dict(batch, is_weight=w))
    eng.step()
    plain = eng_mod.LearnerEngine(eng_mod.PathConfig(**{**cfg.__dict__, "is_exponent": 0.0}))
    plain.load_state_dicts(actor, critic)
    plain.set_batch(batch)
    plain.step()
    torch.cuda.synchronize()
    assert torch.equal(eng.td_sq, plain.td_sq) and torch.equal(eng.priority, plain.priority)
    ref = oracle_for(cfg, actor, critic).iteration(dict(batch, is_weight=w))
    errs = {"q": rel_l2(eng.q_value.cpu().numpy(), ref["q_value"]),
            "target": rel_l2(eng.target_q_value.cpu().numpy(), ref["target_q_value"]),
            "prio": rel_l2(eng.priority.cpu().numpy(), ref["priority"]),
            "critic_loss": abs(eng.losses[0].item() - ref["critic_loss"]) / abs(ref["critic_loss"]),
            "actor_loss": abs(eng.losses[1].item() - ref["actor_loss"]) / abs(ref["actor_loss"])}
    for net in ("actor", "critic"):
        gr = {k: v.cpu().numpy() for k, v in eng.views(net, "grads").items()}
        pa = {k: v.cpu().numpy() for k, v in eng.views(net).items()}
        for k in eng_mod.PARAM_KEYS:
            errs[f"{net}_grad/{k}"] = rel_l2(gr[k], ref[f"{net}_grad"][k])
            errs[f"{net}_after/{k}"] = rel_l2(pa[k], ref[f"{net}_after"][k])
    # dq and the loss of the ABI twin on the oracle's q / q_next
    from r2d2_b200 import native as nv
    L, B, A = cfg.learning, cfg.batch, cfg.act
    f = lambda x: torch.as_tensor(np.ascontiguousarray(x, np.float32)).cuda()  # noqa: E731
    q, qn = f(ref["q_value"].reshape(L, B, A)), f(ref["q_next"])
    T = cfg.rows
    rew, term, wt = f(np.asarray(batch["rew"]).reshape(T, B)), f(np.asarray(batch["term"]).reshape(T, B)), f(w)
    target, dq, loss = torch.empty_like(q), torch.empty_like(q), torch.empty(1, device="cuda")
    td_sq, prio = torch.empty(L * B, device="cuda"), torch.empty(B, device="cuda")
    P = nv.dptr
    nv.check(nv.lib().r2d2_td_priority_weighted(P(q), P(qn), P(rew), P(term), P(wt), L, B, A, cfg.burn_in, cfg.n_step,
                                                cfg.gamma, cfg.eta, P(target), P(dq), P(td_sq), P(prio), P(loss),
                                                nv.current_stream()))
    _, loss_ref, dq_ref, _, _ = lo.td_targets_and_priorities(ref["q_value"].reshape(L, B, A), ref["q_next"],
                                                             np.asarray(batch["rew"], np.float64).reshape(T, B),
                                                             np.asarray(batch["term"], np.float64).reshape(T, B),
                                                             burn_in=cfg.burn_in, learning=L, n_step=cfg.n_step,
                                                             gamma=cfg.gamma, is_weight=w)
    torch.cuda.synchronize()
    errs["dq"] = rel_l2(dq.cpu().numpy(), dq_ref)
    errs["abi_loss"] = abs(loss.item() - loss_ref) / abs(loss_ref)
    bad = {k: v for k, v in errs.items() if not v < TOL}
    assert not bad, bad
    return max(errs.values())


@pytest.mark.parametrize("name", ["ref_pend_h128.npz", "ref_walker_h128.npz"])
def test_weighted_iteration_against_oracle_on_goldens(eng_mod, name):
    kw, actor, critic, batches = golden_case(name)
    cfg = eng_mod.PathConfig(**kw, is_exponent=0.6)
    w = np.random.default_rng(17).uniform(0.05, 1.0, cfg.batch).astype(np.float32)
    worst = _check_weighted_iteration(eng_mod, cfg, actor, critic, batches[0], w)
    print(f"{name} weighted: worst relative error {worst:.3e}")


def test_weighted_iteration_against_oracle_cfg2(eng_mod):
    kw = dict(obs=17, act=6, hidden=256, batch=256, burn_in=40, learning=80, n_step=5)
    actor, critic, batches = port_case(kw, n_batches=1)
    w = np.random.default_rng(19).uniform(0.05, 1.0, 256).astype(np.float32)
    worst = _check_weighted_iteration(eng_mod, eng_mod.PathConfig(**kw, is_exponent=0.6), actor, critic, batches[0], w)
    print(f"cfg-2 weighted: worst relative error {worst:.3e}")


# ---------------------------------------------------------------------------------------------------- 6. pipelining
def test_pipelined_weighted_run_matches_sequential(eng_mod):
    """The weights of batch i+1 come from the prefetch hook, after batch i's priorities are written back - as in the
    sequential sample -> step -> write-back loop.  Eight steps cross two hard target updates."""
    kw = dict(obs=6, act=2, hidden=64, batch=16, burn_in=4, learning=6, n_step=2, target_interval=3)
    cfg = eng_mod.PathConfig(**kw, priority_exponent=0.9, is_exponent=0.6)
    steps = 8

    def shard():
        rng = np.random.default_rng(31)
        rp = eng_mod.DeviceReplay(cfg, capacity_rows=8000)
        rp.add_episodes([episode(rng, cfg, int(rng.integers(30, 90))) for _ in range(50)])
        return rp, torch.Generator(device="cuda").manual_seed(12)

    rp, gen = shard()
    seq = eng_mod.LearnerEngine(cfg, seed=3)
    s_prio, s_w, s_leaf = [], [], []
    for _ in range(steps):
        rp.sample_into(seq, generator=gen)
        s_w.append(seq.is_weight.clone())
        s_leaf.append(seq.leaf_idx.clone())
        seq.step()
        s_prio.append(seq.priority.clone())
        rp.update_priorities(seq.leaf_idx, seq.priority)
    rp2, gen2 = shard()
    pip = eng_mod.LearnerEngine(cfg, seed=3)
    p_prio, p_w, p_leaf = [], [], []

    def hook(e, used):
        p_prio.append(used.priority.clone())
        p_w.append(used.is_weight.clone())
        p_leaf.append(used.leaf_idx.clone())
        rp2.update_priorities(used.leaf_idx, used.priority)
        rp2.sample_into(e, generator=gen2)

    rp2.sample_into(pip, generator=gen2)
    for _ in range(steps):
        pip.step(prefetch=hook)
    torch.cuda.synchronize()
    assert len(p_prio) == steps and pip.step_count == seq.step_count == steps
    assert any((w < 1).any() for w in s_w)
    for it in range(steps):
        assert torch.equal(p_leaf[it], s_leaf[it]), it
        assert rel_l2(p_w[it].cpu().numpy(), s_w[it].cpu().numpy()) < 1e-6, it
        assert rel_l2(p_prio[it].cpu().numpy(), s_prio[it].cpu().numpy()) < 1e-5, it
    for net in ("actor", "critic", "target_actor", "target_critic"):
        assert rel_l2(pip.flat[net].cpu().numpy(), seq.flat[net].cpu().numpy()) < 1e-5, net
    for l in range(rp.stats()["tree_levels"]):
        assert rel_l2(rp.tree_level(l).cpu().numpy(), rp2.tree_level(l).cpu().numpy()) < 1e-5


# ---------------------------------------------------------------------------------------------------- 7. drop-in
def test_dropin_learner_with_prioritized_replay(monkeypatch):
    with trained_dropin_learner(monkeypatch, R2D2_PRIORITY_EXPONENT="0.9", R2D2_IS_EXPONENT="0.6") as (lr, _):
        assert lr.engine.importance_weighting and lr.engine.cfg.is_exponent == 0.6
        w = lr.engine.is_weight.cpu().numpy()
        assert (w > 0).all() and (w <= 1).all() and w.max() == 1.0
        p00 = lr.memory.priority[0][0]                                    # the stored leaf, p^alpha
        assert np.isfinite(p00) and p00 >= 0
        lr.memory.priority[0][0] = 0.25                                   # a raw write is raised on the way in
        torch.cuda.synchronize()
        assert abs(lr.memory.priority[0][0] / 0.25 ** 0.9 - 1) < 1e-6
        out = lr.memory.sample()
        assert len(out) == 10


# ---------------------------------------------------------------------------------------------------- 8. two GPUs
def test_two_gpu_weighted_replicas_stay_identical():
    assert_two_gpu_replicas_stay_identical(dict(SMALL, priority_exponent=0.9, is_exponent=0.6))

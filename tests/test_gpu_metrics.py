"""Learner metrics on the GPU (csrc/metrics.cu, r2d2_b200.metrics): off changes nothing, on changes no training bit, every
field against float64 numpy of the same device tensors, determinism, the data-parallel read rule and the overrun, and
the files the drop-in learner, Actor and ActorPool write."""
import csv
import math
import os

import numpy as np
import pytest
import torch

from learner_harness import SMALL, assert_same_bits, replay_fed_run, trained_dropin_learner
from oracle import ref_port
from peer_harness import PeerGroup, split_batch

pytestmark = pytest.mark.gpu

E = pytest.importorskip("r2d2_b200.engine")
from r2d2_b200 import metrics as M  # noqa: E402
from r2d2_b200 import native as nv  # noqa: E402

# launches metrics add per iteration: the two reduction kernels, and the norm kernel before each Adam without clipping
ADDED_LAUNCHES = {False: 4, True: 2}       # keyed on "clipping on"
ALL_ON = dict(twin_critic=True, is_exponent=0.6, value_rescaling="invertible", grad_clip_norm=0.5)


def _reading(store):
    """replay_fed_run setup: read the metrics once, right before the run closes the engine."""
    def setup(eng):
        close = eng.close

        def close_after_read():
            if "rec" not in store and eng.metrics is not None:
                store["rec"] = eng.metrics.read()
            close()
        eng.close = close_after_read
    return setup


def _mu(eng):
    """The actor head's output mu [L*B*A] in the learner's arena: learner_create carves q, q_next, target, dq, mu one
    after the other, each rounded up to 64 floats."""
    c = eng.cfg
    n = c.learning * c.batch * c.act
    stride = -(-n // 64) * 64
    q = eng.q_value.data_ptr()
    assert eng.target_q_value.data_ptr() == q + 4 * 2 * stride          # the carve order this relies on
    return nv.view_f32(q + 4 * 4 * stride, (n,), eng.device)


def _f64(t):
    return t.detach().cpu().numpy().astype(np.float64).ravel()


def test_off_runs_todays_launches_and_bits():
    lib = nv.lib()
    plain = replay_fed_run(E, 4)
    nulled = replay_fed_run(E, 4, setup=lambda e: nv.check(lib.r2d2_learner_set_metrics(e._h, None, 0)))
    assert int(plain["launches"]) == int(nulled["launches"])
    assert_same_bits(plain, nulled)


@pytest.mark.parametrize("opts", [{}, ALL_ON], ids=["defaults", "twin_beta_rescaling_clip"])
def test_on_changes_no_training_bit(opts):
    off = replay_fed_run(E, 8, **opts)
    store = {}
    on = replay_fed_run(E, 8, setup=_reading(store), metrics=True, **opts)
    clip = opts.get("grad_clip_norm", 0.0) > 0
    assert int(on.pop("launches")) == int(off.pop("launches")) + ADDED_LAUNCHES[clip]
    if not clip:                   # metrics run the norm kernel without clipping: grad_norms is written, Adam is not
        off.pop("grad_norms")
        on.pop("grad_norms")
    assert_same_bits(off, on)
    rec = store["rec"]
    assert rec["iteration"].tolist() == list(range(8))
    assert np.all(np.diff(rec["t_ns"]) > 0)
    assert np.all(np.isfinite(rec["actor_grad_norm"])) and np.all(rec["nonfinite"] == 0)


def test_two_seeded_runs_write_identical_records():
    recs = []
    for _ in range(2):
        store = {}
        replay_fed_run(E, 8, setup=_reading(store), metrics=True, twin_critic=True)
        recs.append(store["rec"])
    for k in recs[0]:
        if k != "t_ns":
            assert np.array_equal(recs[0][k], recs[1][k], equal_nan=True), k


def _one_step(batch_edit=None, actor_scale=None, **extra):
    """A SMALL engine with metrics after one sequential step on a synthetic batch with importance weights."""
    cfg = E.PathConfig(**dict(SMALL, metrics=True, is_exponent=0.5, **extra))
    eng = E.LearnerEngine(cfg, seed=3)
    if actor_scale is not None:
        sd = {k: v.clone() for k, v in eng.views("actor").items()}
        sd["l3.weight"] *= actor_scale
        eng.load_state_dicts(sd, None)
    pc = ref_port.PathConfig(**SMALL)
    batch = ref_port.synthetic_batch(pc, seed=21)
    batch["is_weight"] = np.random.default_rng(4).uniform(0.2, 1.0, SMALL["batch"]).astype(np.float32)
    if batch_edit is not None:
        batch_edit(batch)
    eng.set_batch(batch)
    eng.step()
    torch.cuda.synchronize()
    rec = {k: v[0] for k, v in eng.metrics.read().items()}
    return eng, rec, batch


def _rel(a, b):
    return abs(a - b) / max(abs(b), 1e-300)


@pytest.mark.parametrize("twin", [False, True], ids=["single", "twin"])
def test_fields_match_float64(twin):
    eng, rec, batch = _one_step(twin_critic=twin, grad_clip_norm=1e30)
    q, y, pr, w = _f64(eng.q_value), _f64(eng.target_q_value), _f64(eng.priority), batch["is_weight"].astype(np.float64)
    mu, losses = _f64(_mu(eng)), _f64(eng.losses)
    td = np.abs(q - y)
    assert rec["iteration"] == 0
    means = {"q_mean": q.mean(), "target_mean": y.mean(), "td_abs_mean": td.mean(), "priority_mean": pr.mean(),
             "is_weight_mean": w.mean(), "mu_abs_mean": np.abs(mu).mean()}
    exact = {"q_min": q.min(), "q_max": q.max(), "target_min": y.min(), "target_max": y.max(), "td_abs_max": td.max(),
             "priority_max": pr.max(), "is_weight_min": w.min(), "nonfinite": 0.0,
             "mu_saturated": np.count_nonzero(np.abs(mu) >= np.float32(0.99)) / mu.size,
             "critic_loss": losses[0], "actor_loss": losses[1]}
    if twin:
        means["q2_mean"] = _f64(eng.q_value2).mean()
        exact["critic2_loss"] = losses[2]
    else:
        assert math.isnan(rec["q2_mean"]) and math.isnan(rec["critic2_loss"])
    bad = {k: (rec[k], v) for k, v in means.items() if not _rel(rec[k], v) < 1e-12}
    bad.update({k: (rec[k], v) for k, v in exact.items() if rec[k] != v})
    # clipping on at a bound that never clips: the norms are grad_norms, bit for bit
    gn = eng.grad_norms.cpu().numpy().astype(np.float64)
    bad.update({k: (rec[k], gn[i]) for i, k in enumerate(("critic_grad_norm", "actor_grad_norm")) if rec[k] != gn[i]})
    assert not bad, bad
    eng.close()


def test_grad_norms_without_clipping_match_float64():
    eng, rec, _ = _one_step()
    for net in ("critic", "actor"):
        own = np.sqrt(np.sum(np.square(eng.grads[net].cpu().numpy().astype(np.float64))))   # grad_scale 1
        assert abs(rec[net + "_grad_norm"] / own - 1.0) < 1e-6, net
    eng.close()


def test_weights_off_report_one():
    cfg = E.PathConfig(**dict(SMALL, metrics=True))
    eng = E.LearnerEngine(cfg, seed=3)
    eng.set_batch(ref_port.synthetic_batch(ref_port.PathConfig(**SMALL), seed=2))
    eng.step()
    rec = eng.metrics.read()
    assert rec["is_weight_min"][0] == 1.0 and rec["is_weight_mean"][0] == 1.0
    eng.close()


def test_nonfinite_counts_injected_values():
    Bn = SMALL["burn_in"]

    def poison(batch):
        batch["obs"][Bn + 2, 1, 0] = np.nan            # q of element 1 from row 2 of the window on, and its mu
        batch["rew"][Bn + 3, 5] = np.inf               # the target of element 5 at one step

    eng, rec, _ = _one_step(batch_edit=poison)
    vals = [_f64(eng.q_value), _f64(eng.target_q_value), _f64(_mu(eng))]
    want = sum(int(np.count_nonzero(~np.isfinite(v))) for v in vals)
    assert want > 0 and rec["nonfinite"] == want
    q = vals[0]
    assert rec["q_min"] == np.nanmin(q) and rec["q_max"] == np.nanmax(q)     # min / max skip NaN
    eng.close()


def test_mu_saturated_on_a_saturating_actor():
    eng, rec, _ = _one_step(actor_scale=3000.0)
    mu = _f64(_mu(eng))
    frac = np.count_nonzero(np.abs(mu) >= np.float32(0.99)) / mu.size
    assert frac > 0.5 and rec["mu_saturated"] == frac
    eng.close()


def test_set_metrics_arguments_and_state():
    lib = nv.lib()
    eng = E.LearnerEngine(E.PathConfig(**SMALL), seed=3)
    ring = torch.zeros(int(lib.r2d2_metrics_ring_bytes(4)) // 8 + 1, dtype=torch.float64, device="cuda")
    assert lib.r2d2_learner_set_metrics(eng._h, nv.dptr(ring, torch.float64), 0) == -2       # R2D2_ERR_ARG
    eng.set_batch(ref_port.synthetic_batch(ref_port.PathConfig(**SMALL), seed=2))
    eng.step()
    assert lib.r2d2_learner_set_metrics(eng._h, nv.dptr(ring, torch.float64), 4) == -4       # R2D2_ERR_STATE
    eng.close()


# ------------------------------------------------------------------------------------------------ data parallel
def _dp_batches(n, world):
    pc = ref_port.PathConfig(**dict(SMALL, batch=SMALL["batch"] * world))
    return [split_batch(ref_port.synthetic_batch(pc, seed=60 + i), world) for i in range(n)]


def test_data_parallel_read_rule():
    g = PeerGroup(2, dict(SMALL, metrics=True))
    seen = []

    def on_iteration(it):
        recs = [e.metrics.read() for e in g.engines]
        # the finish phase of iteration it - 1 ran after critic phase it: its record, actor norm included, is readable
        want = [] if it == 0 else [it - 1]
        for r in recs:
            assert r["iteration"].tolist() == want
            assert np.all(np.isfinite(r["actor_grad_norm"]))
        for k in ("critic_grad_norm", "actor_grad_norm"):
            assert np.array_equal(recs[0][k], recs[1][k]), k
        seen.extend(want)

    try:
        g.run(_dp_batches(4, 2), on_iteration=on_iteration)
        recs = [e.metrics.read() for e in g.engines]
        assert [r["iteration"].tolist() for r in recs] == [[3], [3]]
        assert recs[0]["actor_grad_norm"][0] == recs[1]["actor_grad_norm"][0]
        assert seen == [0, 1, 2]
        g.check_status()
    finally:
        g.close()


def test_data_parallel_ring_overrun():
    g = PeerGroup(2, dict(SMALL))
    try:
        readers = [M.LearnerMetrics.attach(e, slots=2) for e in g.engines]
        g.run(_dp_batches(4, 2))
        for m in readers:
            with pytest.raises(RuntimeError, match="iteration 2 overwrote iteration 0"):
                m.read()
        g.check_status()
    finally:
        g.close()


# ------------------------------------------------------------------------------------------------ drop-in files
def _csv(path):
    with open(path) as f:
        return list(csv.DictReader(f))


def test_dropin_learner_writes_one_row_per_step(monkeypatch):
    with trained_dropin_learner(monkeypatch, R2D2_METRICS="1") as (lr, actors):
        rows = _csv("model_data/metrics/learner_rank0.csv")
        assert [int(r["iteration"]) for r in rows] == [0, 1, 2, 3]
        assert list(rows[0]) == list(M.field_names())
        assert all(math.isfinite(float(r["critic_grad_norm"])) and math.isfinite(float(r["actor_grad_norm"]))
                   for r in rows)
        for a in actors:
            ep = _csv("model_data/metrics/episodes_actor%d.csv" % a.actor_id)
            assert [int(r["episode"]) for r in ep] == [1, 2, 3, 4, 5]
            assert all(int(r["actor_id"]) == a.actor_id and int(r["kept"]) == 1 for r in ep)


def test_dropin_learner_without_metrics_writes_no_directory(monkeypatch):
    with trained_dropin_learner(monkeypatch, R2D2_METRICS="0") as (lr, _):
        assert lr.engine.metrics is None
        assert not os.path.exists("model_data/metrics")


def test_actor_pool_episode_rows_match_its_returns(monkeypatch, tmp_path):
    from actor_pool import ActorPool
    for k, v in dict(R2D2_OBS_SIZE="5", R2D2_N_ACTIONS="2", R2D2_HIDDEN="64", R2D2_METRICS="1").items():
        monkeypatch.setenv(k, v)
    monkeypatch.chdir(tmp_path)
    os.makedirs("memory_data")
    os.makedirs("model_data")
    pool = ActorPool([4, 5, 6], device="cuda", noise_std=0.1, seed=3)
    for env, n in zip(pool.envs, (70, 45, 90)):
        env.episode_len = n                 # lane 1 finishes episodes shorter than 60 steps: not kept
    returns = {}
    finish = pool._finish_episodes

    def record(lanes):
        for lane in lanes:
            returns[(pool.actor_ids[lane], pool.episode[lane])] = (pool.reward_sum[lane], len(pool.sequence[lane]))
        finish(lanes)
    pool._finish_episodes = record
    pool.run(max_steps=200)
    rows = _csv("model_data/metrics/episodes_pool4.csv")
    assert len(rows) == len(returns) >= 6
    for r in rows:
        ret, length = returns[(int(r["actor_id"]), int(r["episode"]))]
        assert float(r["return"]) == ret and int(r["length"]) == length
        assert int(r["kept"]) == int(length >= 60)
    assert {int(r["kept"]) for r in rows} == {0, 1}

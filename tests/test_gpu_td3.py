"""TD3's target on the GPU: the defaults keep their bits and launches, a twin whose critics are equal behaves like one
critic, the smoothing kernel's noise against the numpy Philox restatement, multi-iteration runs against the float64
TD3 oracle (goldens, cfg-2, rescaling with importance weights, A = 1 and 64), the pipelined / replay-fed / resumed
schedules bit for bit, the data-parallel exchange of the doubled critic block on one GPU, and the drop-in learner."""
import os

import numpy as np
import pytest
import torch

from conftest import rel_l2
from learner_harness import (SMALL, TOL, assert_pipelined_matches_sequential, assert_resumed_run_is_bit_identical,
                             assert_same_bits, assert_two_gpu_replicas_stay_identical, check_against_oracle, fixed_run,
                             golden_case, oracle_for, port_case, replay_fed_run, trained_dropin_learner)
from oracle import ref_port
from oracle import target_noise as tn
from peer_harness import PeerGroup, split_batch

pytestmark = pytest.mark.gpu

TD3 = dict(twin_critic=True, target_noise=0.2, target_noise_clip=0.5)


@pytest.fixture(scope="module")
def E():
    from r2d2_b200 import engine
    return engine


def _np(sd):
    return {k: v.detach().cpu().numpy() for k, v in sd.items()}


# ---------------------------------------------------------------------------------------------------- 1. defaults
def test_defaults_keep_bits_and_launches(E):
    base = fixed_run(E)
    assert_same_bits(base, fixed_run(E, twin_critic=False, target_noise=0.0))
    assert_same_bits(base, fixed_run(E, setter=lambda e: e.set_target_smoothing(0.0, 0.5, 0, 0)))
    twin = fixed_run(E, twin_critic=True)
    smooth = fixed_run(E, **TD3)
    assert int(smooth["launches"]) == int(twin["launches"]) + 1 > int(base["launches"])   # one smoothing launch
    assert fixed_run(E, target_noise=0.2)["launches"] == base["launches"] + 1


def test_library_rejects_bad_values(E):
    eng = E.LearnerEngine(E.PathConfig(**SMALL))
    lib = eng.lib
    for sigma, clip in ((-0.1, 0.5), (float("nan"), 0.5), (float("inf"), 0.5), (0.2, 0.0), (0.2, -1.0),
                        (0.2, float("inf")), (0.2, float("nan"))):
        assert lib.r2d2_learner_set_target_smoothing(eng._h, sigma, clip, 0, 0) == -2          # R2D2_ERR_ARG
    assert lib.r2d2_learner_set_target_smoothing(eng._h, 0.2, 0.5, 0, 0) == 0
    pc = ref_port.PathConfig(**SMALL)
    eng.set_batch(ref_port.synthetic_batch(pc, seed=1))
    eng.step(prefetch=lambda e, used: e.set_batch(ref_port.synthetic_batch(pc, seed=2)))   # next targets run ahead
    assert lib.r2d2_learner_set_target_smoothing(eng._h, 0.1, 0.5, 0, 0) == -4              # R2D2_ERR_STATE
    eng.step()
    assert lib.r2d2_learner_set_target_smoothing(eng._h, 0.1, 0.5, 0, 0) == 0
    from r2d2_b200 import native as nv
    bad = nv.LearnerOptions(2)
    h = nv.c_void_p()
    assert lib.r2d2_learner_create_ex(nv.byref(h), nv.byref(nv.LearnerConfig()), nv.byref(bad)) == -2
    eng.close()


def test_twin_memory_is_reported(E):
    a = E.LearnerEngine(E.PathConfig(**SMALL))
    b = E.LearnerEngine(E.PathConfig(**SMALL, twin_critic=True))
    assert a.twin_added_bytes == 0 and b.twin_added_bytes > 0 and a.q_value2 is None
    P = a.flat["critic"].numel()
    assert b._critic2_off % 64 == 0 and P <= b._critic2_off < P + 64 and b.flat["critic"].numel() == 2 * b._critic2_off
    assert len(b.losses) == 3
    a.close()
    b.close()


# ---------------------------------------------------------------------------------------------------- 2. symmetry
def test_equal_twins_behave_like_one_critic(E):
    pc = ref_port.PathConfig(**SMALL)
    batch = ref_port.synthetic_batch(pc, seed=5)
    batch["c_state"][:] = 0
    batch["tc_state"][:] = 0
    twin = E.LearnerEngine(E.PathConfig(**SMALL, twin_critic=True), seed=4)
    one = E.LearnerEngine(E.PathConfig(**SMALL), seed=4)
    twin.load_state_dicts(None, None, critic2=twin.state_dict("critic"), target_critic2=twin.state_dict("target_critic"))
    for e in (twin, one):
        e.set_batch(batch)
        e.step()
    torch.cuda.synchronize()
    P, off = twin._n_critic, twin._critic2_off
    assert torch.equal(twin.q_value2, twin.q_value)
    assert torch.equal(twin.losses[2], twin.losses[0])
    g = twin.grads["critic"]
    assert torch.equal(g[:P], g[off:off + P]) and not g[P:off].any() and not g[off + P:].any()
    assert torch.equal(twin.target_q_value, one.target_q_value)
    assert torch.equal(twin.q_value, one.q_value) and torch.equal(twin.priority, one.priority)
    twin.close()
    one.close()


# ---------------------------------------------------------------------------------------------------- 3. noise
def _device_z(lib, n, seed, rank, it):
    """r2d2_target_smoothing on mu = 0 with sigma = 2^-4: every |sigma z| < 1, so out * 16 is z exactly."""
    from r2d2_b200 import native as nv
    mu = torch.zeros(n, device="cuda")
    out = torch.empty_like(mu)
    nv.check(lib.r2d2_target_smoothing(nv.dptr(mu), nv.dptr(out), n, 0.0625, 1e30, seed, rank, it, nv.current_stream()))
    torch.cuda.synchronize()
    return out.cpu().numpy().astype(np.float64) * 16.0


def test_noise_matches_numpy_philox(E):
    from r2d2_b200 import native as nv
    lib = nv.lib()
    n = (1 << 20) + 3                                    # a partial last group of four
    for seed, rank, it in ((0, 0, 0), (12345, 3, 7), (2 ** 32 - 1, 1, 2 ** 33 + 5)):
        got, want = _device_z(lib, n, seed, rank, it), tn.normal(n, seed, rank, it)
        err = np.abs(got - want) / np.maximum(np.abs(want), 1e-30)
        assert err.max() < 1e-6, (seed, rank, it, float(err.max()))
    base = _device_z(lib, 4096, 5, 0, 1)
    for other in (_device_z(lib, 4096, 5, 1, 1), _device_z(lib, 4096, 5, 0, 2), _device_z(lib, 4096, 6, 0, 1)):
        assert not np.any(other == base)
    from scipy import stats
    res = stats.kstest(_device_z(lib, 1 << 20, 2024, 0, 0), "norm")     # fixed seed: deterministic
    assert res.pvalue > 1e-3, res


def test_noise_clip_and_final_clamp(E):
    from r2d2_b200 import native as nv
    lib = nv.lib()
    n = 1 << 16
    mu = torch.full((n,), 0.9, device="cuda")
    out = torch.empty_like(mu)
    nv.check(lib.r2d2_target_smoothing(nv.dptr(mu), nv.dptr(out), n, 1.0, 0.3, 9, 0, 4, nv.current_stream()))
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    low = np.float32(np.float32(0.9) - np.float32(0.3))
    assert got.max() == 1.0 and got.min() == low and (got == low).sum() > 100 and (got == 1.0).sum() > 100
    want = tn.smooth(np.full(n, np.float32(0.9), np.float64), 1.0, float(np.float32(0.3)), 9, 0, 4)
    assert np.abs(got - want).max() < 1e-6


# ---------------------------------------------------------------------------------------------------- 4. float64
SETTINGS = {"smooth": dict(TD3), "smooth_polyak_clip": dict(TD3, target_tau=0.005, target_interval=1)}


@pytest.mark.parametrize("setting", sorted(SETTINGS))
@pytest.mark.parametrize("name", ["ref_pend_h128.npz", "ref_walker_h128.npz"])
def test_runs_against_oracle_on_goldens(E, name, setting):
    kw, actor, critic, batches = golden_case(name)
    worst = check_against_oracle(E, dict(kw, **SETTINGS[setting]), actor, critic, batches, 12,
                                 probe_clip=setting == "smooth_polyak_clip")
    print(f"{name} {setting}: worst relative error {worst:.3e}")


def test_runs_against_oracle_cfg2(E):
    kw = dict(obs=17, act=6, hidden=256, batch=256, burn_in=40, learning=80, n_step=5)
    print(f"cfg-2: worst relative error {check_against_oracle(E, dict(kw, **TD3), *port_case(kw), 6):.3e}")


def test_rescaling_and_importance_weights_against_oracle(E):
    kw = dict(obs=11, act=3, hidden=128, batch=32, burn_in=10, learning=20, n_step=3)
    w = np.random.default_rng(3).uniform(0.2, 1.0, kw["batch"]).astype(np.float32)
    w[0] = 1.0
    extra = dict(TD3, value_rescaling="invertible", rescaling_eps=1e-3, is_exponent=0.6)
    worst = check_against_oracle(E, dict(kw, **extra), *port_case(kw), 6, weights=lambda it: w)
    print(f"invertible + IS weights: worst relative error {worst:.3e}")


@pytest.mark.parametrize("act", [1, 64])
def test_action_widths_through_the_smoothing_kernel(E, act):
    kw = dict(obs=7, act=act, hidden=64, batch=16, burn_in=4, learning=8, n_step=2)
    print(f"A={act}: worst relative error {check_against_oracle(E, dict(kw, **TD3), *port_case(kw), 4):.3e}")


# ---------------------------------------------------------------------------------------------------- 5. schedules
SCHED = dict(TD3, target_tau=0.3, target_interval=3, grad_clip_norm=0.05)


def test_pipelined_step_matches_sequential_bit_for_bit(E):
    """Interval 3: on two of three iterations the next batch's target chains (and their noise) run ahead."""
    assert_pipelined_matches_sequential(E, E.PathConfig(**SMALL, **SCHED), 7)


def test_replay_fed_runs_are_bitwise_reproducible(E):
    assert_same_bits(replay_fed_run(E, 7, **SCHED), replay_fed_run(E, 7, **SCHED))


def test_resumed_run_is_bit_identical(E):
    def check_state(st):
        assert {"critic2", "target_critic2", "critic2_optimizer"} <= set(st) and st["twin_critic"] is True
    assert_resumed_run_is_bit_identical(E, E.PathConfig(**SMALL, **SCHED), check_state)


# ---------------------------------------------------------------------------------------------------- 6. data parallel
DP = dict(obs=6, act=2, hidden=64, batch=8, burn_in=4, learning=6, n_step=2, target_interval=2)


def test_dp_identical_shards_without_noise_give_the_single_engine_bits(E):
    pc = ref_port.PathConfig(**{k: v for k, v in DP.items() if k != "target_interval"})
    batches = [ref_port.synthetic_batch(pc, seed=60 + i) for i in range(4)]
    one = E.LearnerEngine(E.PathConfig(**DP, twin_critic=True), seed=2)
    for b in batches:
        one.set_batch(b)
        one.step()
    grp = PeerGroup(2, dict(DP, twin_critic=True), seed=2)
    grp.run([[b, b] for b in batches])
    grp.flush()
    grp.check_status()
    torch.cuda.synchronize()
    for r, eng in enumerate(grp.engines):
        for net in ("actor", "critic", "target_actor", "target_critic"):
            assert torch.equal(eng.flat[net], one.flat[net]), (r, net)
        for d in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(getattr(eng, d)["critic"], getattr(one, d)["critic"]), (r, d)
    grp.close()
    one.close()


def test_dp_disjoint_shards_with_rank_keyed_noise_against_oracle(E):
    kw = dict(DP, batch=16)
    pc = ref_port.PathConfig(**{k: v for k, v in kw.items() if k != "target_interval"})
    batches = [ref_port.synthetic_batch(pc, seed=80 + i) for i in range(5)]
    grp = PeerGroup(2, dict(kw, batch=kw["batch"] // 2, **TD3), seed=2)     # every rank one half of the global batch
    for r, eng in enumerate(grp.engines):
        eng.set_target_smoothing(rank=r)
    e0 = grp.engines[0]
    ol = oracle_for(e0.cfg, _np(e0.views("actor")), _np(e0.views("critic")), _np(e0.views("critic2")))
    shards = [split_batch(b, 2) for b in batches]
    grp.run(shards)
    grp.flush()
    grp.check_status()
    for s in shards:
        ol.iteration(s)
    errs = {}
    for net in ("actor", "critic", "critic2", "target_actor", "target_critic", "target_critic2"):
        for k, v in e0.views(net).items():
            errs[f"{net}/{k}"] = rel_l2(v.cpu().numpy(), getattr(ol, net)[k])
    grp.close()
    bad = {k: v for k, v in errs.items() if not v < TOL}
    assert not bad, bad


# ---------------------------------------------------------------------------------------------------- 7. drop-in
def test_dropin_learner_with_td3(monkeypatch):
    with trained_dropin_learner(monkeypatch, R2D2_TWIN_CRITIC="1", R2D2_TARGET_NOISE="0.2", R2D2_TARGET_NOISE_CLIP="0.5",
                                R2D2_TARGET_NOISE_SEED="3", R2D2_TARGET_TAU="0.005",
                                R2D2_TARGET_INTERVAL="1") as (lr, _):
        c = lr.engine.cfg
        assert (c.twin_critic, c.target_noise, c.target_noise_clip, c.target_noise_seed) == (True, 0.2, 0.5, 3)
        assert len(lr.engine.losses) == 3
        md = torch.load(os.path.join("model_data", "model.pt"), map_location="cpu")
        assert sorted(md) == ["actor", "critic", "target_actor", "target_critic"]
        assert md["critic"]["l3.bias"].numel() == 2 and lr.engine.flat["critic"].numel() == 2 * lr.engine._critic2_off
        lr.update_target_model()
        assert torch.equal(lr.engine.flat["target_critic"], lr.engine.flat["critic"])


# ---------------------------------------------------------------------------------------------------- 8. two GPUs
def test_two_gpu_replicas_stay_identical_with_td3():
    assert_two_gpu_replicas_stay_identical(dict(SMALL, **SCHED))

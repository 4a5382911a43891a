"""Optimiser-step extras on the GPU: the Polyak target update fused into the Adam launches (target_tau) and per-net
global gradient-norm clipping (grad_clip_norm) - against torch's soft_update bit for bit, against the float64 oracle
over multi-iteration runs, the defaults against the plain path, and the pipelined / resumed / repeated schedules against
each other."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from learner_harness import (SMALL, assert_pipelined_matches_sequential, assert_resumed_run_is_bit_identical,
                             assert_same_bits, assert_two_gpu_replicas_stay_identical, check_against_oracle, fixed_run,
                             golden_case, port_case, replay_fed_run, trained_dropin_learner)
from oracle import ref_port

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng_mod():
    from r2d2_b200 import engine
    return engine


# ---------------------------------------------------------------------------------------------------- 1. torch parity
def test_polyak_update_is_torch_soft_update_bit_for_bit(eng_mod):
    """One update iteration: each target equals utils.soft_update, run by torch on the same device tensors with the
    float32 value of tau, applied to the targets before the step and the post-step weights."""
    import utils
    tau = float(np.float32(0.005))
    cfg = eng_mod.PathConfig(**SMALL, target_tau=0.005, target_interval=1)
    eng = eng_mod.LearnerEngine(cfg, seed=2)
    g = torch.Generator().manual_seed(5)
    for n in ("target_actor", "target_critic"):                 # targets that differ from the nets
        eng.flat[n].add_(0.01 * torch.randn(eng.flat[n].shape, generator=g).to(eng.device))
    before = {n: eng.flat[n].clone() for n in ("target_actor", "target_critic")}
    eng.set_batch(ref_port.synthetic_batch(ref_port.PathConfig(**SMALL), seed=1))
    eng.step()
    torch.cuda.synchronize()
    for net in ("actor", "critic"):
        want = SimpleNamespace(parameters=lambda t=before["target_" + net]: [t])
        utils.soft_update(want, SimpleNamespace(parameters=lambda p=eng.flat[net]: [p]), tau)
        assert torch.equal(eng.flat["target_" + net], before["target_" + net]), net
        assert not torch.equal(eng.flat["target_" + net], eng.flat[net])


# ---------------------------------------------------------------------------------------------------- 2. float64 oracle
@pytest.mark.parametrize("tau,interval", [(0.05, 1), (0.3, 3)])
@pytest.mark.parametrize("name", ["ref_pend_h128.npz", "ref_walker_h128.npz"])
def test_runs_against_oracle_on_goldens(eng_mod, name, tau, interval):
    """Clipping at a tenth of the first norm; q / target / priority from the second iteration on, when the engine runs
    on updated weights and targets."""
    kw, actor, critic, batches = golden_case(name)
    worst = check_against_oracle(eng_mod, dict(kw, target_tau=tau, target_interval=interval), actor, critic, batches, 12,
                                 first=1, probe_clip=True, norms=True)
    print(f"{name} tau={tau} interval={interval}: worst relative error {worst:.3e}")


@pytest.mark.parametrize("tau,interval", [(0.05, 1), (0.3, 3)])
def test_runs_against_oracle_cfg2(eng_mod, tau, interval):
    kw = dict(obs=17, act=6, hidden=256, batch=256, burn_in=40, learning=80, n_step=5)
    worst = check_against_oracle(eng_mod, dict(kw, target_tau=tau, target_interval=interval), *port_case(kw), 6,
                                 first=1, probe_clip=True, norms=True)
    print(f"cfg-2 tau={tau} interval={interval}: worst relative error {worst:.3e}")


# ---------------------------------------------------------------------------------------------------- 3. defaults
def test_clip_bound_that_never_clips_keeps_the_unclipped_bits(eng_mod):
    off, big = fixed_run(eng_mod), fixed_run(eng_mod, grad_clip_norm=1e30)
    assert big.pop("launches") == off.pop("launches") + 2           # one norm kernel per net
    norms = big.pop("grad_norms")
    assert (norms > 0).all() and torch.equal(off.pop("grad_norms"), torch.zeros_like(norms))   # off: nothing computed
    assert_same_bits(off, big)


def test_default_launch_count_is_unchanged(eng_mod):
    base = fixed_run(eng_mod)["launches"]
    assert fixed_run(eng_mod, target_tau=1.0, grad_clip_norm=0.0)["launches"] == base
    assert fixed_run(eng_mod, target_tau=0.5)["launches"] == base          # the blend rides on the Adam launches
    assert fixed_run(eng_mod, grad_clip_norm=0.01)["launches"] == base + 2


def test_library_rejects_bad_values(eng_mod):
    eng = eng_mod.LearnerEngine(eng_mod.PathConfig(**SMALL))
    lib = eng.lib
    for tau in (0.0, -0.5, 1.0001, float("nan"), float("inf")):
        assert lib.r2d2_learner_set_target_tau(eng._h, tau) == -2                # R2D2_ERR_ARG
    for m in (-1.0, float("nan"), float("inf")):
        assert lib.r2d2_learner_set_grad_clip(eng._h, m) == -2
    assert lib.r2d2_learner_set_target_tau(eng._h, 1.0) == 0 and lib.r2d2_learner_set_grad_clip(eng._h, 0.0) == 0
    eng.close()


# ---------------------------------------------------------------------------------------------------- 4. schedules
def test_pipelined_step_matches_sequential_bit_for_bit(eng_mod):
    """At interval 1 every iteration updates the targets, so the pipelined step never runs the next target chains
    ahead and calls the hook at the end: the same kernels in the same order as the sequential loop."""
    cfg = eng_mod.PathConfig(**SMALL, target_tau=0.05, target_interval=1, grad_clip_norm=0.01)
    a = assert_pipelined_matches_sequential(eng_mod, cfg, 6)
    assert (a["grad_norms"] > 0.01).any()


def test_replay_fed_runs_are_bitwise_reproducible(eng_mod):
    """Interval 3: the next batch's target chains run ahead on two of three iterations and wait on the third."""
    kw = dict(target_tau=0.3, target_interval=3, grad_clip_norm=0.05)
    a = replay_fed_run(eng_mod, 7, **kw)
    assert_same_bits(a, replay_fed_run(eng_mod, 7, **kw))
    assert not torch.equal(a["flat.target_critic"], a["flat.critic"])


def test_resumed_run_is_bit_identical(eng_mod):
    """Crosses the Polyak updates at steps 3 and 6."""
    assert_resumed_run_is_bit_identical(eng_mod, eng_mod.PathConfig(**SMALL, target_tau=0.3, target_interval=3,
                                                                     grad_clip_norm=0.05))


# ---------------------------------------------------------------------------------------------------- 5. drop-in
def test_dropin_learner_with_soft_targets_and_clipping(monkeypatch):
    with trained_dropin_learner(monkeypatch, R2D2_TARGET_TAU="0.05", R2D2_TARGET_INTERVAL="1",
                                R2D2_GRAD_CLIP="0.5") as (lr, _):
        c = lr.engine.cfg
        assert (c.target_tau, c.target_interval, c.grad_clip_norm) == (0.05, 1, 0.5)
        norms = lr.engine.grad_norms.cpu().numpy()
        assert np.isfinite(norms).all() and (norms > 0).all()
        for net in ("actor", "critic"):                      # soft targets: neither the old nets nor a copy
            assert not torch.equal(lr.engine.flat["target_" + net], lr.engine.flat[net])


# ---------------------------------------------------------------------------------------------------- 6. two GPUs
def test_two_gpu_replicas_stay_identical_with_clipping_and_polyak():
    assert_two_gpu_replicas_stay_identical(dict(SMALL, target_tau=0.05, target_interval=1, grad_clip_norm=0.05))

"""Optimiser-step extras on the host side: the float64 oracle's target_tau and grad_clip against torch's own
clip_grad_norm_ + Adam + soft_update on float64 modules, PathConfig and drop-in validation, and the compiler's report
on the new kernels (no spills, no local memory)."""
import numpy as np
import pytest
import torch

from learner_harness import fake_engine_learner
from oracle import learner_oracle as lo
from oracle import ref_port
from sass_report import functions, library_sass, ops, ptxas_report


@pytest.mark.parametrize("tau,interval,clip", [(0.05, 1, 0.1), (0.3, 3, 0.0), (1.0, 2, 1e9), (0.5, 2, 1e-4)])
def test_oracle_matches_torch_clip_adam_soft_update(tau, interval, clip):
    """Six iterations of the float64 torch port of the reference learner with clip_grad_norm_ before each Adam step and
    utils.soft_update on the update iterations, against the oracle with target_tau and grad_clip."""
    import utils
    kw = dict(obs=4, act=2, hidden=8, batch=3, burn_in=2, learning=3, n_step=2)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        port = ref_port.PortLearner(ref_port.PathConfig(**kw, target_interval=1 << 30), seed=4)
        sd = lambda m: {k: v.detach().numpy().copy() for k, v in m.state_dict().items()}  # noqa: E731
        ol = lo.OracleLearner(sd(port.actor), sd(port.critic), burn_in=2, learning=3, n_step=2,
                              target_interval=interval, target_tau=tau, grad_clip=clip)
        torch_norms, clipped = {}, False
        for net, opt in (("critic", port.critic_opt), ("actor", port.actor_opt)):
            params = list(getattr(port, net).parameters())

            def step(orig=opt.step, params=params, net=net):
                torch_norms[net] = float(torch.nn.utils.clip_grad_norm_(params, clip if clip > 0 else float("inf")))
                return orig()
            opt.step = step
        for it in range(6):
            batch = {k: np.asarray(v, np.float64) for k, v in ref_port.synthetic_batch(port.cfg, seed=10 + it).items()}
            port.iteration(batch)
            if (it + 1) % interval == 0:
                utils.soft_update(port.target_actor, port.actor, tau)
                utils.soft_update(port.target_critic, port.critic, tau)
            ol.iteration(batch)
            for net in ("critic", "actor"):
                assert abs(ol.norms[net] / torch_norms[net] - 1) < 1e-12, (it, net)
                clipped |= 0 < clip < ol.norms[net]
        rel = lambda a, b: np.linalg.norm(a - b) / np.linalg.norm(b)  # noqa: E731
        for net in ("actor", "critic", "target_actor", "target_critic"):
            got, want = getattr(ol, net), sd(getattr(port, net))
            for k in lo.PARAM_KEYS:
                assert rel(got[k], want[k]) < 1e-10, (net, k)
        for net, opt in (("actor", port.actor_opt), ("critic", port.critic_opt)):
            st = getattr(ol, net + "_adam")
            for k, p in getattr(port, net).named_parameters():
                assert rel(st["m/" + k], opt.state[p]["exp_avg"].numpy()) < 1e-10, (net, k)
                assert rel(st["v/" + k], opt.state[p]["exp_avg_sq"].numpy()) < 1e-10, (net, k)
        assert clipped == (0 < clip < 1e9)                                     # the clipping arms do clip
    finally:
        torch.set_default_dtype(prev)


def test_path_config_optimiser_values_are_validated():
    from r2d2_b200 import engine
    cfg = engine.PathConfig(obs=3, act=1)
    assert (cfg.target_tau, cfg.grad_clip_norm) == (1.0, 0.0)          # the reference's hard copy, no clipping
    engine.PathConfig(obs=3, act=1, target_tau=0.005, target_interval=1, grad_clip_norm=10.0)
    for bad in ({"target_tau": 0.0}, {"target_tau": 1.5}, {"target_tau": -0.1}, {"target_tau": float("nan")},
                {"grad_clip_norm": -1.0}, {"grad_clip_norm": float("inf")}, {"grad_clip_norm": float("nan")}):
        with pytest.raises(ValueError):
            engine.PathConfig(obs=3, act=1, **bad)


def test_dropin_optimiser_environment_variables(monkeypatch, tmp_path):
    lr = fake_engine_learner(monkeypatch, tmp_path, R2D2_TARGET_TAU="0.005", R2D2_TARGET_INTERVAL="1", R2D2_GRAD_CLIP="40")
    c = lr.engine.cfg
    assert (c.target_tau, c.target_interval, c.grad_clip_norm) == (0.005, 1, 40.0)
    for k in ("R2D2_TARGET_TAU", "R2D2_TARGET_INTERVAL", "R2D2_GRAD_CLIP"):
        monkeypatch.delenv(k)
    c = fake_engine_learner(monkeypatch, tmp_path).engine.cfg
    assert (c.target_tau, c.target_interval, c.grad_clip_norm) == (1.0, 500, 0.0)
    for bad in (dict(R2D2_TARGET_TAU="0"), dict(R2D2_TARGET_TAU="2"), dict(R2D2_GRAD_CLIP="-1"),
                dict(R2D2_TARGET_INTERVAL="0")):
        with pytest.raises(ValueError):
            fake_engine_learner(monkeypatch, tmp_path, **bad)
        monkeypatch.delenv(next(iter(bad)))


NEW_KERNELS = ("adam_kernel", "grad_norm_kernel")


def test_optimiser_kernels_do_not_spill():
    report, stderr = ptxas_report("elementwise.cu")
    found = {k: 0 for k in NEW_KERNELS}
    for m in report:
        for k in NEW_KERNELS:
            if k in m.group(1):
                found[k] += 1
                assert m.group(2) == m.group(3) == m.group(4) == "0", m.group(0)
    assert found == {"adam_kernel": 4, "grad_norm_kernel": 1}, stderr[-2000:]


def test_optimiser_sass_has_no_local_memory():
    sass = library_sass()
    for k, want in (("adam_kernel", 4), ("grad_norm_kernel", 1)):
        funcs = functions(sass, k)
        assert len(funcs) == want, sorted(funcs)
        for name, body in funcs.items():
            body_ops = [op for op, _ in ops(body)]
            assert not [op for op in body_ops if op.startswith(("LDL", "STL"))], f"local-memory traffic in {name}"
    # the fused Polyak update rounds like torch: FMUL, FMUL, FADD - the blend is never contracted into an FFMA
    for name, body in functions(sass, "adam_kernel").items():
        if "ILb0ELb1E" in name or "ILb1ELb1E" in name:
            body_ops = [op for op, _ in ops(body)]
            assert body_ops.count("FADD") >= 1 and body_ops.count("FMUL") >= 2, name

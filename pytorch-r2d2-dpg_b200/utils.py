"""Drop-in for the reference's utils.py (same names and argument meaning, utils.py:4-21).

Host-side helpers only: inside the learner these formulas run fused in the CUDA TD/priority kernel
(csrc/elementwise.cu); the functions here serve the actor side and code that mixes reference and new pieces.
"""
import numpy as np
import torch


def soft_update(target_model, model, tau):
    """Polyak update theta' <- (1-tau) theta' + tau theta (utils.py:4-6).  Two rounded products and one rounded add, as
    the reference computes it and as the learner's fused update (PathConfig.target_tau) rounds it."""
    with torch.no_grad():
        for tp, p in zip(target_model.parameters(), model.parameters()):
            tp.copy_(tp * (1.0 - tau) + p * tau)


def get_obs(observation):
    """Flatten a dm_control observation dict into a [1, obs] float32 array (utils.py:8-15)."""
    parts = [np.ravel(np.asarray(v, dtype=np.float32)) for v in observation.values()]
    return np.concatenate(parts).astype(np.float32)[None, :]


def calc_priority(td_loss, eta=0.9):
    """eta * max + (1 - eta) * mean of a window of squared TD values (utils.py:17-18)."""
    vals = list(td_loss)
    return eta * max(vals) + (1.0 - eta) * (sum(vals) / len(vals))


def value_rescale(x, eps=1e-3):
    """R2D2's h_eps(x) = sign(x) (sqrt(|x| + 1) - 1) + eps x, as sign(x) |x| / (sqrt(|x| + 1) + 1) + eps x: the same
    function without the cancellation of sqrt(|x| + 1) - 1 near 0 (the form the learner's TD kernels use)."""
    a = torch.abs(x)
    return torch.sign(x) * (a / (torch.sqrt(a + 1) + 1)) + eps * x


def inverse_value_rescale(x, eps=1e-3):
    """h_eps^-1(x) = sign(x) v (v + 2), v = 2|x| / ((1 + 2 eps) + sqrt((1 + 2 eps)^2 + 4 eps |x|)), the positive root of
    eps v^2 + (1 + 2 eps) v - |x| = 0; no step cancels, and eps = 0 gives (|x| + 1)^2 - 1."""
    a = torch.abs(x)
    c = 1.0 + 2.0 * eps
    v = 2 * a / (c + torch.sqrt(c * c + 4 * eps * a))
    return torch.sign(x) * (v * (v + 2))


def invertical_vf(x):
    """Value rescaling h(x) = sign(x) (sqrt(|x| + 1) - 1) without the eps*x term (utils.py:20-21)."""
    return torch.sign(x) * (torch.sqrt(torch.abs(x) + 1) - 1)

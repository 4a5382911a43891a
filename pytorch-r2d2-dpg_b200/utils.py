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


def invertical_vf(x):
    """Value rescaling h(x) = sign(x) (sqrt(|x| + 1) - 1) without the eps*x term (utils.py:20-21)."""
    return torch.sign(x) * (torch.sqrt(torch.abs(x) + 1) - 1)

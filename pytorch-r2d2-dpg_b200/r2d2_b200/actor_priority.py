"""Actor-side rows of the path on the GPU (SURVEY 8f N2): the n-step reward pre-sum and the initial sequence
priorities that every reference actor computes per finished episode at batch 1 on its own nets
(reference actor.py:74-76 `calc_nstep_reward`, :78-107 `calc_priorities`), batched over episodes:

    B = episodes, time-major zero-padded rows -> three persistent chains from the zero state
    (online critic on the stored actions, target actor, target critic on the target actor's actions:
    r2d2_lstm_net_forward, the learner's own kernels) -> r2d2_actor_priorities (windowed TD kernel).

The reference's quirks are kept (see include/r2d2_b200.h): every net sees rows 0, 1, 2, ... once; the deque of
`learning` TD values is one step ahead of the learner's window; the TD is the mean difference over actions, squared.
With R2D2's options (r2d2_b200.td_options) the target is h_eps(R + gamma^n (1-d) h_eps^-1(Q')) and/or the priority is
taken over |td| (still the mean difference over actions) instead of td^2.
"""
from __future__ import annotations

import numpy as np
import torch

from . import native as nv
from . import td_options

PARAM_KEYS = ("l1.weight", "l1.bias", "l2.weight_ih", "l2.weight_hh", "l2.bias_ih", "l2.bias_hh", "l3.weight", "l3.bias")


def _flat(sd, device):
    return torch.cat([torch.as_tensor(np.asarray(sd[k]) if not isinstance(sd[k], torch.Tensor) else sd[k],
                                      dtype=torch.float32).reshape(-1) for k in PARAM_KEYS]).to(device).contiguous()


def nstep_rewards(raw_tb: torch.Tensor, n_rows: torch.Tensor, n_step: int, gamma: float) -> torch.Tensor:
    """raw_tb [T,B] float32 CUDA (time-major, one episode per column), n_rows [B] int32 rows incl. pad rows."""
    out = torch.empty_like(raw_tb)
    T, B = raw_tb.shape
    nv.check(nv.lib().r2d2_nstep_rewards(nv.dptr(raw_tb), nv.dptr(n_rows, torch.int32), T, B, n_step, gamma, nv.dptr(out),
                                         nv.current_stream()))
    return out


def episode_priorities(critic, target_actor, target_critic, episodes, *, hidden, burn_in=20, learning=40, n_step=5,
                       gamma=0.997, eta=0.9, rewards_are_raw=False, device=None, rescaling="reference",
                       eps=td_options.DEFAULT_EPS, priority_metric="squared", obs_norm=None):
    """episodes: list of (obs [N,O], act [N,A], rew [N], term [N]) host arrays, N = real rows + n_step pad rows
    (actor.py:173).  Weights: state_dicts (or dicts of arrays) with the reference's keys.  rescaling / eps /
    priority_metric: r2d2_b200.td_options (the defaults are the reference's).  obs_norm: model.pt's `obs_norm` entry
    {mean_f, inv_std_f, clip} - the chains then read the normalised observations (r2d2_obs_normalize) - or None.  Returns
    (list of float32 arrays [N - n_step - burn_in - learning], list of n-step reward arrays [N])."""
    opts = td_options.TdOptions(rescaling, eps, priority_metric)
    if not torch.cuda.is_available():
        raise nv.NativeError("episode_priorities needs a CUDA device; there is no CPU fallback")
    lib = nv.lib()
    dev = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
    B = len(episodes)
    O, A = episodes[0][0].shape[1], episodes[0][1].shape[1]
    lens = [int(e[0].shape[0]) for e in episodes]
    T = max(lens)
    obs = torch.zeros((T, B, O), dtype=torch.float32)
    act = torch.zeros((T, B, A), dtype=torch.float32)
    rew = torch.zeros((T, B), dtype=torch.float32)
    term = torch.ones((T, B), dtype=torch.float32)
    for b, (o, a, r, d) in enumerate(episodes):
        n = lens[b]
        obs[:n, b] = torch.as_tensor(np.asarray(o, np.float32))
        act[:n, b] = torch.as_tensor(np.asarray(a, np.float32))
        rew[:n, b] = torch.as_tensor(np.asarray(r, np.float32).reshape(-1))
        term[:n, b] = torch.as_tensor(np.asarray(d, np.float32).reshape(-1))
    obs, act, rew, term = (x.to(dev) for x in (obs, act, rew, term))
    n_rows = torch.tensor(lens, dtype=torch.int32, device=dev)
    if obs_norm is not None:
        mean_f = torch.as_tensor(obs_norm["mean_f"], dtype=torch.float32).to(dev).contiguous()
        inv_std_f = torch.as_tensor(obs_norm["inv_std_f"], dtype=torch.float32).to(dev).contiguous()
        nv.check(lib.r2d2_obs_normalize(nv.dptr(obs), nv.dptr(obs), T * B, O, nv.dptr(mean_f), nv.dptr(inv_std_f),
                                        float(obs_norm["clip"]), nv.current_stream()))
    if rewards_are_raw:
        rew = nstep_rewards(rew, n_rows, n_step, gamma)
    st = nv.current_stream()
    sh_c, sh_a = nv.NetShape(O, A, hidden, 1), nv.NetShape(O, A, hidden, 0)
    Te = T - n_step                                        # the online critic stops n_step rows early (actor.py:91)
    ws = torch.empty(max(lib.r2d2_net_workspace_floats(nv.byref(sh_c), T, B, 1),
                         lib.r2d2_net_workspace_floats(nv.byref(sh_a), T, B, 1)), device=dev)
    p_c, p_ta, p_tc = _flat(critic, dev), _flat(target_actor, dev), _flat(target_critic, dev)
    q = torch.empty((Te, B, A), device=dev)
    a_t = torch.empty((T, B, A), device=dev)
    q_t = torch.empty((T, B, A), device=dev)
    nv.check(lib.r2d2_lstm_net_forward(nv.byref(sh_c), nv.dptr(p_c), nv.dptr(obs), nv.dptr(act), None, None, Te, B, 1, 0,
                                       nv.dptr(q), nv.dptr(ws), st))
    nv.check(lib.r2d2_lstm_net_forward(nv.byref(sh_a), nv.dptr(p_ta), nv.dptr(obs), None, None, None, T, B, 1, 0,
                                       nv.dptr(a_t), nv.dptr(ws), st))
    nv.check(lib.r2d2_lstm_net_forward(nv.byref(sh_c), nv.dptr(p_tc), nv.dptr(obs), nv.dptr(a_t), None, None, T, B, 1, 0,
                                       nv.dptr(q_t), nv.dptr(ws), st))
    p_max = max(1, Te - (burn_in + learning))
    prio = torch.empty((B, p_max), device=dev)
    if opts.is_default:
        nv.check(lib.r2d2_actor_priorities(nv.dptr(q), nv.dptr(q_t), nv.dptr(rew), nv.dptr(term),
                                           nv.dptr(n_rows, torch.int32), B, A, burn_in, learning, n_step, gamma, eta, p_max,
                                           nv.dptr(prio), st))
    else:
        nv.check(lib.r2d2_actor_priorities_ex(nv.dptr(q), nv.dptr(q_t), nv.dptr(rew), nv.dptr(term),
                                              nv.dptr(n_rows, torch.int32), B, A, burn_in, learning, n_step, gamma, eta,
                                              p_max, nv.dptr(prio), nv.byref(nv.TdOptions(*opts.native())), st))
    prio_h, rew_h = prio.cpu().numpy(), rew.cpu().numpy()
    out = [prio_h[b, :max(0, lens[b] - n_step - burn_in - learning)].copy() for b in range(B)]
    return out, [rew_h[:lens[b], b].copy() for b in range(B)]

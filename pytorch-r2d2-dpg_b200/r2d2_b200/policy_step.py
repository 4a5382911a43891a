"""Actor side, per env step: the four recurrent nets of N actor lanes stepped once on the GPU (r2d2_policy_step,
csrc/policy.cu), the batched form of what every reference actor does on the CPU at batch 1 (actor.py:149-154):

    action = actor(x); critic(x, action); target_critic(x, target_actor(x))

`PolicyStepper` keeps the four flat parameter blocks and a ring of recurrent states on the device.  Per env step the
only host<->device traffic is obs in and mu out (and, with exploration set, the actions); an episode's state history
crosses PCIe once, when it is read back with `episode_states`.

With `set_exploration` (r2d2_b200.exploration, gaussian or ou) the step kernel also draws each lane's exploration noise
from its actor id and the step count, and `actions` holds the noisy actions of the last step.
"""
from __future__ import annotations

from ctypes import c_void_p

import numpy as np
import torch

from . import native as nv
from .actor_priority import _flat

NETS = ("actor", "target_actor", "critic", "target_critic")   # the replay's state order (actor.py:149,166)


def policy_step(params, obs, state_in, state_out, mu, workspace=None, obs_norm=None, exploration=None, action=None):
    """One step on CUDA tensors: params = 4 flat blocks (NETS order), obs [N,O], state_in / state_out [4,2,N,H],
    mu [N,A] (written).  obs_norm: (mean_f [O], inv_std_f [O] CUDA tensors, clip) - the nets read the normalised obs
    (r2d2_policy_step_ex) - or None.  exploration: dict(mode="gaussian"|"ou", seed, step, one_minus_theta, actor_id
    [N] int32, sigma [N], ou_state [N,A] or None) with CUDA tensors, and action [N,A] (written): r2d2_policy_step_explore,
    which synchronises the stream once to check sigma.  Otherwise launches on the current stream and does not
    synchronise."""
    N, O = obs.shape
    A, H = mu.shape[1], state_in.shape[3]
    lib = nv.lib()
    shape = nv.NetShape(O, A, H, 0)
    if workspace is None:
        workspace = torch.empty(max(1, lib.r2d2_policy_workspace_floats(nv.byref(shape), N)), device=obs.device)
    ptrs = (c_void_p * 4)(*[nv.dptr(p).value for p in params])
    if exploration is not None:
        e = exploration
        mean_f, inv_std_f, clip = obs_norm if obs_norm is not None else (None, None, 0.0)
        ex = nv.Exploration(nv.EXPLORATION_OU if e["mode"] == "ou" else nv.EXPLORATION_GAUSSIAN, int(e["seed"]),
                            int(e["step"]), float(e["one_minus_theta"]), nv.dptr(e["actor_id"], torch.int32),
                            nv.dptr(e["sigma"]), nv.dptr(e.get("ou_state")))
        nv.check(lib.r2d2_policy_step_explore(nv.byref(shape), ptrs, nv.dptr(obs), nv.dptr(state_in),
                                              nv.dptr(state_out), nv.dptr(mu), N, nv.dptr(workspace), nv.dptr(mean_f),
                                              nv.dptr(inv_std_f), float(clip), nv.byref(ex), nv.dptr(action),
                                              nv.current_stream()))
    elif obs_norm is None:
        nv.check(lib.r2d2_policy_step(nv.byref(shape), ptrs, nv.dptr(obs), nv.dptr(state_in), nv.dptr(state_out),
                                      nv.dptr(mu), N, nv.dptr(workspace), nv.current_stream()))
    else:
        mean_f, inv_std_f, clip = obs_norm
        nv.check(lib.r2d2_policy_step_ex(nv.byref(shape), ptrs, nv.dptr(obs), nv.dptr(state_in), nv.dptr(state_out),
                                         nv.dptr(mu), N, nv.dptr(workspace), nv.dptr(mean_f), nv.dptr(inv_std_f),
                                         float(clip), nv.current_stream()))


class StateRing:
    """Recurrent state history of N lanes: `ring[(M + 1), 4, 2, N, H]`, where pool step k reads slot k mod (M + 1) and
    writes slot k + 1.  A lane's episode that began at step `start[lane]` keeps its states while it has at most
    M = max_episode_steps steps.  Subclasses implement `load(model_dict)`, `_step(obs, state_in, state_out)` and
    `set_exploration(options, actor_ids)`; the noise of a step is drawn at t = `self.t` (the steps taken before it),
    and `reset` zeroes the lanes' OU state."""

    def __init__(self, obs_size, n_actions, hidden, n_lanes, device, max_episode_steps):
        self.obs_size, self.n_actions, self.hidden, self.n_lanes = obs_size, n_actions, hidden, n_lanes
        self.max_episode_steps = int(max_episode_steps)
        self.device = torch.device(device)
        self.ring = torch.zeros((self.max_episode_steps + 1, 4, 2, n_lanes, hidden), device=self.device)
        self.t = 0                                   # steps taken so far
        self.start = np.zeros(n_lanes, np.int64)    # step at which each lane's current episode began
        self.actions = None                          # with exploration set: the last step's actions [N,A] float32

    def _slot(self, k):
        return k % (self.max_episode_steps + 1)

    def reset(self, lanes):
        """Zero state for these lanes (models.py:34-36); their episodes begin at the next step."""
        s = self._slot(self.t)
        for lane in lanes:
            self.ring[s, :, :, lane].zero_()
            self.start[lane] = self.t

    def current_states(self):
        """[4,2,N,H] view of the states the next step reads."""
        return self.ring[self._slot(self.t)]

    def step(self, obs):
        """obs [N,O] host array -> mu [N,A] host array (the actor's output before exploration noise; with exploration
        set, `actions` then holds this step's noisy actions)."""
        long_lanes = np.nonzero(self.t - self.start + 1 > self.max_episode_steps)[0]
        if len(long_lanes):
            raise RuntimeError("episode of lane %d has outgrown max_episode_steps=%d: raise max_episode_steps"
                               % (int(long_lanes[0]), self.max_episode_steps))
        mu = self._step(obs, self.ring[self._slot(self.t)], self.ring[self._slot(self.t + 1)])
        self.t += 1
        return mu

    def episode_states(self, lane, first, last):
        """States of `lane` before steps first .. last-1 -> host float32 [last - first, 4, 2, H]."""
        if not (self.start[lane] <= first <= last <= self.t):
            raise ValueError("steps [%d, %d) are not in lane %d's current episode [%d, %d)"
                             % (first, last, lane, int(self.start[lane]), self.t))
        a, n = self._slot(first), last - first
        if a + n <= self.max_episode_steps + 1:
            st = self.ring[a:a + n, :, :, lane]
        else:
            st = torch.cat((self.ring[a:, :, :, lane], self.ring[:a + n - self.max_episode_steps - 1, :, :, lane]))
        return st.to("cpu", copy=True).numpy()           # never a view of the ring (a CPU ring is reused)


class PolicyStepper(StateRing):
    """r2d2_policy_step for n_lanes lanes on one GPU, with pinned obs / mu staging buffers."""

    def __init__(self, obs_size, n_actions, hidden, n_lanes, device=None, max_episode_steps=1000):
        if not torch.cuda.is_available():
            raise nv.NativeError("PolicyStepper needs a CUDA device; there is no CPU fallback")
        dev = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        super().__init__(obs_size, n_actions, hidden, n_lanes, dev, max_episode_steps)
        lib = nv.lib()
        counts = [lib.r2d2_net_param_count(nv.byref(nv.NetShape(obs_size, n_actions, hidden, int(k >= 2))))
                  for k in range(4)]
        self.params = [torch.zeros(c, device=dev) for c in counts]
        shape = nv.NetShape(obs_size, n_actions, hidden, 0)
        self.workspace = torch.empty(lib.r2d2_policy_workspace_floats(nv.byref(shape), n_lanes), device=dev)
        self.obs_host = torch.empty((n_lanes, obs_size), pin_memory=True)
        self.mu_host = torch.empty((n_lanes, n_actions), pin_memory=True)
        self.obs_dev = torch.empty((n_lanes, obs_size), device=dev)
        self.mu_dev = torch.empty((n_lanes, n_actions), device=dev)
        self.obs_norm = None          # (mean_f, inv_std_f, clip) on the device from model.pt's `obs_norm`, or None
        self.exploration = None       # set_exploration: the r2d2_exploration fields and device arrays

    def load(self, model_dict):
        """model.pt dict {'actor', 'target_actor', 'critic', 'target_critic'} -> the four flat blocks (plain copies).
        An `obs_norm` entry {mean_f, inv_std_f, clip} makes every later step read normalised obs; without it raw obs."""
        for p, name in zip(self.params, NETS):
            flat = _flat(model_dict[name], self.device)
            if flat.numel() != p.numel():
                raise ValueError("%s: %d parameters, the stepper was built for %d" % (name, flat.numel(), p.numel()))
            p.copy_(flat)
        n = model_dict.get("obs_norm")
        self.obs_norm = None if n is None else (
            torch.as_tensor(n["mean_f"], dtype=torch.float32).to(self.device).contiguous(),
            torch.as_tensor(n["inv_std_f"], dtype=torch.float32).to(self.device).contiguous(), float(n["clip"]))

    def set_exploration(self, options, actor_ids):
        """Draw exploration noise in the step (options: r2d2_b200.exploration.Exploration, gaussian or ou) for lane k
        = actor id actor_ids[k]: the ids and sigma_i are uploaded once; the OU state starts at zero."""
        if options.mode not in ("gaussian", "ou"):
            raise ValueError("set_exploration: mode %r draws no noise in the step" % (options.mode,))
        ids = list(actor_ids)
        if len(ids) != self.n_lanes:
            raise ValueError("set_exploration: %d actor ids for %d lanes" % (len(ids), self.n_lanes))
        sigma = options.sigmas(ids)                  # validates the ids against the schedule
        if max(ids) >= 2 ** 31:
            raise ValueError("set_exploration: actor ids must be < 2**31")
        dev = self.device
        self.exploration = dict(
            mode=options.mode, seed=options.seed, one_minus_theta=float(options.one_minus_theta),
            actor_id=torch.tensor(ids, dtype=torch.int32, device=dev), sigma=torch.from_numpy(sigma).to(dev),
            ou_state=torch.zeros((self.n_lanes, self.n_actions), device=dev) if options.mode == "ou" else None)
        self.action_host = torch.empty((self.n_lanes, self.n_actions), pin_memory=True)
        self.action_dev = torch.empty((self.n_lanes, self.n_actions), device=dev)

    def reset(self, lanes):
        lanes = list(lanes)
        super().reset(lanes)
        if self.exploration is not None and self.exploration["ou_state"] is not None and lanes:
            self.exploration["ou_state"][torch.as_tensor(lanes, device=self.device)] = 0.0

    def _step(self, obs, state_in, state_out):
        self.obs_host.numpy()[:] = obs
        with torch.cuda.device(self.device):
            self.obs_dev.copy_(self.obs_host, non_blocking=True)
            if self.exploration is None:
                policy_step(self.params, self.obs_dev, state_in, state_out, self.mu_dev, self.workspace, self.obs_norm)
            else:
                policy_step(self.params, self.obs_dev, state_in, state_out, self.mu_dev, self.workspace, self.obs_norm,
                            exploration=dict(self.exploration, step=self.t), action=self.action_dev)
                self.action_host.copy_(self.action_dev, non_blocking=True)
            self.mu_host.copy_(self.mu_dev, non_blocking=True)
            torch.cuda.current_stream().synchronize()
        if self.exploration is not None:
            self.actions = self.action_host.numpy().copy()
        return self.mu_host.numpy().copy()

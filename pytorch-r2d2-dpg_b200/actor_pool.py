"""Many reference actors in one process: `ActorPool(actor_ids)` runs one lane per actor id and steps the four
recurrent nets of all lanes together on the GPU (r2d2_b200.policy_step.PolicyStepper -> r2d2_policy_step), while each
lane steps its own environment on the host.  Lane by lane it does what `Actor.run` does (actor.py:138-179):

  * env from `actor._make_env(actor_id)`, action repeat 4; action = clip(mu + N(0, noise_std), -1, 1), or under
    R2D2_EXPLORATION=gaussian|ou (r2d2_b200.exploration) the actions the stepper draws for each lane's actor id at
    t = the pool step, the noise a drop-in Actor with that id draws at its own step t;
  * the recorded recurrent state of a step is the state BEFORE that step, nets in the order actor, target_actor,
    critic, target_critic (actor.py:149,166);
  * episodes shorter than burn_in + learning = 60 steps are dropped; kept ones get n_step pad rows, n-step rewards and
    initial priorities (r2d2_b200.actor_priority.episode_priorities, batched over every lane that finished on the same
    step), with the target / priority options of the environment (r2d2_b200.td_options, as the learner reads them);
  * each lane has its own ReplayMemory, saved to memory{actor_id}.pt once it holds more than 3 episodes (same file
    format and atomic rename);
  * model.pt is reloaded every 500 pool steps; lane 0 prints its episode reward;
  * with R2D2_METRICS=1 every lane's finished episodes are appended to ./model_data/metrics/episodes_pool{first actor
    id}.csv (r2d2_b200.metrics: actor id, episode, pool step, length, return, kept).

Differences from separate Actor processes:
  * the lanes step in lock-step: a lane whose episode ends starts the next one on the next pool step;
  * all lanes share one initial weight set until model.pt exists (each Actor draws its own);
  * in the reference exploration mode, the noise comes from one seeded generator per pool, not from each process's
    global numpy state (the gaussian and ou modes key it on the actor id and the step, as Actor does).

`actor_pool_process(actor_ids)` is the process entry point (picklable under spawn); pool_launch.py starts pools next to
the learner.  The stepper and the priority function are arguments so the host bookkeeping can run with
`ModelsStepper`, the models.py nets on any torch device (a reference for tests and measurements, never chosen
automatically).
"""
import os
from copy import deepcopy
from time import perf_counter, sleep

import numpy as np
import torch

from actor import _make_env
from models import ActorNet, CriticNet
from r2d2_b200.policy_step import NETS, StateRing
from replay_memory import ReplayMemory
from utils import get_obs


class ModelsStepper(StateRing):
    """The four models.py nets stepped at batch n_lanes with torch on `device` (the drop-in actor's arithmetic)."""

    def __init__(self, obs_size, n_actions, hidden, n_lanes, device="cpu", max_episode_steps=1000):
        super().__init__(obs_size, n_actions, hidden, n_lanes, device, max_episode_steps)
        self.nets = [cls(obs_size, n_actions, 0, hidden=hidden).to(self.device).eval()
                     for cls in (ActorNet, ActorNet, CriticNet, CriticNet)]
        self.obs_norm = None
        self.noise = None             # set_exploration: r2d2_b200.exploration.HostNoise, the kernel's noise on the host

    def set_exploration(self, options, actor_ids):
        from r2d2_b200.exploration import HostNoise
        if len(actor_ids) != self.n_lanes:
            raise ValueError("set_exploration: %d actor ids for %d lanes" % (len(actor_ids), self.n_lanes))
        self.noise = HostNoise(options, actor_ids, self.n_actions)

    def reset(self, lanes):
        lanes = list(lanes)
        super().reset(lanes)
        if self.noise is not None:
            self.noise.reset(lanes)

    def load(self, model_dict):
        for net, name in zip(self.nets, NETS):
            net.load_state_dict(model_dict[name])
        self.obs_norm = model_dict.get("obs_norm")    # {mean_f, inv_std_f, clip}: the nets read normalised obs

    @torch.no_grad()
    def _step(self, obs, state_in, state_out):
        actor, target_actor, critic, target_critic = self.nets
        for k, net in enumerate(self.nets):
            net.set_state(state_in[k, 0], state_in[k, 1])
        x = torch.as_tensor(np.asarray(obs, np.float32)).to(self.device)
        if self.obs_norm is not None:
            from r2d2_b200.obs_norm import normalize_torch
            n = self.obs_norm
            x = normalize_torch(x, n["mean_f"], n["inv_std_f"], n["clip"])
        mu = actor(x)
        critic(x, mu)
        target_critic(x, target_actor(x))
        for k, net in enumerate(self.nets):
            state_out[k, 0], state_out[k, 1] = net.hx, net.cx
        mu = mu.cpu().numpy()
        if self.noise is not None:
            self.actions = self.noise.actions(mu, self.t)
        return mu


def initial_model_dict(obs_size, n_actions, hidden):
    """One fresh weight set (models.py init), target nets equal to the online nets as in Actor.__init__."""
    a = ActorNet(obs_size, n_actions, 0, hidden=hidden).state_dict()
    c = CriticNet(obs_size, n_actions, 0, hidden=hidden).state_dict()
    return {"actor": a, "target_actor": deepcopy(a), "critic": c, "target_critic": deepcopy(c)}


def actor_pool_process(actor_ids, device=None):
    pool = ActorPool(actor_ids, device=device)
    pool.run()


class ActorPool:
    def __init__(self, actor_ids, device=None, noise_std=0.3, stepper=None, priority_fn=None, seed=0,
                 max_episode_steps=1000):
        self.actor_ids = list(actor_ids)
        self.envs = [_make_env(i) for i in self.actor_ids]
        self.n_lanes = len(self.envs)
        self.action_size = self.envs[0].action_spec().shape[0]
        self.obs_size = get_obs(self.envs[0].reset().observation).shape[1]
        self.burn_in_length, self.learning_length, self.n_step = 20, 40, 5
        self.sequence_length = self.burn_in_length + self.learning_length
        self.memory_sequence_size = 1000
        self.memories = [ReplayMemory(memory_sequence_size=self.memory_sequence_size) for _ in self.actor_ids]
        self.memory_save_interval = 3
        self.gamma = 0.997
        self.actor_parameter_update_interval = 500
        self.model_path = './model_data/'
        self.hidden = int(os.environ.get("R2D2_HIDDEN", 128))
        self.noise_std = noise_std
        self.rng = np.random.default_rng(seed)
        if stepper is None:
            from r2d2_b200.policy_step import PolicyStepper
            stepper = PolicyStepper(self.obs_size, self.action_size, self.hidden, self.n_lanes, device=device,
                                    max_episode_steps=max_episode_steps)
        self.stepper = stepper
        self.device = stepper.device
        from r2d2_b200 import exploration, td_options
        self.td_options = td_options.from_environ()
        self.exploration = exploration.from_environ()
        if self.exploration.mode != "reference":
            self.stepper.set_exploration(self.exploration, self.actor_ids)
        from r2d2_b200 import metrics
        self.episode_log = metrics.episode_csv("pool", self.actor_ids[0]) if metrics.from_environ() else None
        self.priority_fn = priority_fn or self._gpu_priorities
        self.model_dict = initial_model_dict(self.obs_size, self.action_size, self.hidden)
        self.stepper.load(self.model_dict)
        self.load_model()
        self.steps = 0
        self.episode = [0] * self.n_lanes
        self.host_time = self.device_time = 0.0      # seconds spent stepping envs / in stepper.step
        self.obs = np.zeros((self.n_lanes, self.obs_size), np.float32)
        self.sequence = [[] for _ in self.actor_ids]
        self.reward_sum = [0.0] * self.n_lanes
        self.last_mu = None
        self._begin_episodes(range(self.n_lanes))

    def _gpu_priorities(self, model_dict, episodes):
        from r2d2_b200 import actor_priority
        return actor_priority.episode_priorities(
            model_dict["critic"], model_dict["target_actor"], model_dict["target_critic"], episodes,
            hidden=self.hidden, burn_in=self.burn_in_length, learning=self.learning_length, n_step=self.n_step,
            gamma=self.gamma, rewards_are_raw=True, device=self.device, rescaling=self.td_options.value_rescaling,
            eps=self.td_options.rescaling_eps, priority_metric=self.td_options.priority_metric,
            obs_norm=model_dict.get("obs_norm"))

    def load_model(self):
        """Follow the learner's model.pt (actor.py:50-72); retried while the file is being replaced."""
        path = self.model_path + 'model.pt'
        if not os.path.isfile(path):
            return
        for _ in range(20):
            try:
                model_dict = torch.load(path, map_location="cpu")
                self.stepper.load(model_dict)
                self.model_dict = model_dict
                return
            except Exception:
                sleep(np.random.rand() * 2 + 0.5)

    def _begin_episodes(self, lanes):
        lanes = list(lanes)
        for lane in lanes:
            self.obs[lane] = get_obs(self.envs[lane].reset().observation)[0]
            self.sequence[lane] = []
            self.reward_sum[lane] = 0.0
            self.episode[lane] += 1
        self.stepper.reset(lanes)

    def step(self):
        """One env step of every lane."""
        t0 = perf_counter()
        mu = self.stepper.step(self.obs)
        t1 = perf_counter()
        self.last_mu = mu
        if self.exploration.mode == "reference":
            actions = mu + self.rng.normal(0.0, self.noise_std, mu.shape) if self.noise_std else mu
            actions = np.clip(actions, -1, 1)
        else:
            actions = self.stepper.actions
        finished = []
        for lane, env in enumerate(self.envs):
            action = actions[lane]
            reward = 0.0
            for _ in range(4):                                        # action repeat, actor.py:152-157
                time_step = env.step(action)
                next_obs = get_obs(time_step.observation)
                reward += time_step.reward or 0.0
                if time_step.last():
                    break
            self.reward_sum[lane] += reward
            self.sequence[lane].append((self.obs[lane].copy(), action.astype(np.float32), [reward],
                                        [1.0 if time_step.last() else 0.0]))
            self.obs[lane] = next_obs[0]
            if time_step.last():
                finished.append(lane)
        self.steps += 1
        self.device_time += t1 - t0
        self.host_time += perf_counter() - t1
        if self.steps % self.actor_parameter_update_interval == 0:
            self.load_model()
        if finished:
            self._finish_episodes(finished)

    def _finish_episodes(self, lanes):
        kept, log = [], []
        for lane in lanes:
            seq = self.sequence[lane]
            if lane == 0:
                print('episode:', self.episode[0], 'step:', self.steps, 'reward:', self.reward_sum[0])
            log.append((self.actor_ids[lane], self.episode[lane], self.steps, len(seq), self.reward_sum[lane],
                        len(seq) >= self.sequence_length))
            if len(seq) < self.sequence_length:
                continue
            start = int(self.stepper.start[lane])
            states = self.stepper.episode_states(lane, start, start + len(seq))
            pad = [(np.zeros(self.obs_size, np.float32), np.zeros(self.action_size, np.float32), [0.0], [1.0])
                   for _ in range(self.n_step)]
            kept.append((lane, seq + pad, states))
        if kept:
            episodes = [(np.stack([r[0] for r in seq]), np.stack([r[1] for r in seq]),
                         np.asarray([r[2][0] for r in seq], np.float32), np.asarray([r[3][0] for r in seq], np.float32))
                        for _, seq, _ in kept]
            prios, rewards = self.priority_fn(self.model_dict, episodes)
            for (lane, seq, states), prio, rew in zip(kept, prios, rewards):
                rows = [(o, a, [float(rew[i])], d) for i, (o, a, _, d) in enumerate(seq)]
                recurrent = [[[st[k, 0], st[k, 1]] for k in range(4)] for st in states]
                self.memories[lane].add(rows, recurrent, list(prio))
        if self.episode_log is not None:
            from r2d2_b200 import metrics
            metrics.append_csv(self.episode_log, metrics.EPISODE_COLUMNS, log)
        for lane in lanes:
            if len(self.memories[lane].memory) > self.memory_save_interval:
                self.memories[lane].save(self.actor_ids[lane])
        self._begin_episodes(lanes)

    def run(self, max_steps=None):
        """Step until `max_steps` more pool steps have run (forever if None)."""
        end = None if max_steps is None else self.steps + max_steps
        while end is None or self.steps < end:
            self.step()

"""Drop-in for the reference's actor.py: `Actor(actor_id)`, `.run()`, `.load_model()`,
`.calc_nstep_reward()`, `.calc_priorities()`, `actor_process(actor_id)` (actor.py:16-180).

The actor is OUTSIDE the accelerated hot path (SURVEY 8: CPU actors stay as they are); this module
exists so the reference's r2d2.py imports and runs unchanged, and it keeps the episode tuple, recurrent
state and memory{i}.pt formats the learner ingests.  Without dm_control it steps a synthetic
environment of the configured shape (BASELINE.json configs[4]: "Humanoid-shape synthetic env").
"""
import os
from collections import deque
from copy import deepcopy
from time import sleep

import numpy as np
import torch

from models import ActorNet, CriticNet
from r2d2_b200 import exploration
from r2d2_b200 import metrics
from r2d2_b200 import obs_norm as obs_norm_mod
from r2d2_b200 import td_options
from replay_memory import ReplayMemory
from utils import calc_priority, get_obs, inverse_value_rescale, invertical_vf, value_rescale


class _SyntheticEnv:
    """Random linear dynamics with the dm_control TimeStep surface (reset/step/last/observation/reward)."""

    class _TS:
        def __init__(self, obs, reward, last):
            self.observation, self.reward, self._last = {"o": obs}, reward, last

        def last(self):
            return self._last

    def __init__(self, obs_size, n_actions, episode_len=250, seed=0):
        self.rng = np.random.default_rng(seed)
        self.obs_size, self.n_actions, self.episode_len = obs_size, n_actions, episode_len
        self.A = self.rng.standard_normal((obs_size, obs_size)).astype(np.float32) * 0.1
        self.Bm = self.rng.standard_normal((n_actions, obs_size)).astype(np.float32) * 0.5

    def action_spec(self):
        return type("Spec", (), {"shape": (self.n_actions,)})()

    def reset(self):
        self.t = 0
        self.x = self.rng.standard_normal(self.obs_size).astype(np.float32)
        return self._TS(self.x, 0.0, False)

    def step(self, action):
        self.t += 1
        self.x = np.tanh(self.x @ self.A + np.asarray(action, np.float32) @ self.Bm).astype(np.float32)
        return self._TS(self.x, float(-np.square(self.x).mean()), self.t >= self.episode_len * 4)


def _make_env(actor_id):
    if "R2D2_OBS_SIZE" not in os.environ:
        try:
            from dm_control import suite
            return suite.load(domain_name="walker", task_name="run")
        except ImportError:
            pass
    return _SyntheticEnv(int(os.environ.get("R2D2_OBS_SIZE", 24)), int(os.environ.get("R2D2_N_ACTIONS", 6)),
                         seed=actor_id)


def actor_process(actor_id):
    actor = Actor(actor_id)
    actor.run()


class Actor:
    def __init__(self, actor_id):
        self.env = _make_env(actor_id)
        self.action_size = self.env.action_spec().shape[0]
        self.obs_size = get_obs(self.env.reset().observation).shape[1]
        self.actor_id = actor_id
        self.burn_in_length, self.learning_length, self.n_step = 20, 40, 5
        self.sequence_length = self.burn_in_length + self.learning_length
        self.sequence, self.recurrent_state, self.priority = [], [], []
        self.td_loss = deque(maxlen=self.learning_length)
        self.memory_sequence_size = 1000
        self.memory = ReplayMemory(memory_sequence_size=self.memory_sequence_size)
        self.memory_save_interval = 3
        self.gamma = 0.997
        self.actor_parameter_update_interval = 500
        self.model_path = './model_data/'
        self.hidden = int(os.environ.get("R2D2_HIDDEN", 128))
        self.td_options = td_options.from_environ()     # the learner's n-step target / priority options
        self.device = torch.device(os.environ.get("R2D2_ACTOR_DEVICE", "cpu"))  # actors are CPU workers here
        self.actor = ActorNet(self.obs_size, self.action_size, 0, hidden=self.hidden).to(self.device).eval()
        self.target_actor = deepcopy(self.actor)
        self.critic = CriticNet(self.obs_size, self.action_size, 0, hidden=self.hidden).to(self.device).eval()
        self.target_critic = deepcopy(self.critic)
        self.obs_norm = None      # model.pt's `obs_norm` {mean_f, inv_std_f, clip} when the learner normalises obs
        # R2D2_EXPLORATION=gaussian|ou: noise keyed on (seed, actor id, step), as ActorPool lanes and the GPU draw it
        self.exploration = exploration.from_environ()
        self.noise = None if self.exploration.mode == "reference" else \
            exploration.HostNoise(self.exploration, [actor_id], self.action_size)
        # R2D2_METRICS=1: one row per finished episode (r2d2_b200.metrics.EPISODE_COLUMNS)
        self.episode_log = metrics.episode_csv("actor", actor_id) if metrics.from_environ() else None
        self.load_model()

    def _nets(self):
        return (("actor", self.actor), ("target_actor", self.target_actor), ("critic", self.critic),
                ("target_critic", self.target_critic))

    def load_model(self):
        """Follow the learner's model.pt (actor.py:50-72); retried while the file is being replaced."""
        path = self.model_path + 'model.pt'
        if not os.path.isfile(path):
            return
        for _ in range(20):
            try:
                model_dict = torch.load(path, map_location=self.device)
                for name, net in self._nets():
                    net.load_state_dict(model_dict[name])
                self.obs_norm = model_dict.get('obs_norm')
                return
            except Exception:
                sleep(np.random.rand() * 2 + 0.5)

    def _obs(self, x):
        """What the nets read: the raw observation, or its normalised form under the learner's statistics."""
        n = self.obs_norm
        return x if n is None else obs_norm_mod.normalize_torch(x, n['mean_f'], n['inv_std_f'], n['clip'])

    def calc_nstep_reward(self):
        """Overwrite rewards with their n-step discounted sums (actor.py:74-76)."""
        for i in range(len(self.sequence) - self.n_step):
            self.sequence[i][2][0] = sum(self.sequence[i + j][2][0] * (self.gamma ** j) for j in range(self.n_step))

    @torch.no_grad()
    def calc_priorities(self):
        """Initial sequence priorities by replaying the episode through the four nets (actor.py:78-107).  Under R2D2's
        options (r2d2_b200.td_options) the target is h_eps(R + gamma^n (1-d) h_eps^-1(Q')) and the priority is taken over
        |mean difference| instead of its square."""
        opt = self.td_options
        invertible, eps = opt.value_rescaling == "invertible", opt.rescaling_eps
        for _, net in self._nets():
            net.reset_state()
        self.td_loss = deque(maxlen=self.learning_length)
        self.priority = []
        t = lambda a: torch.from_numpy(np.asarray(a, np.float32)).to(self.device).unsqueeze(0)  # noqa: E731
        o = lambda a: self._obs(t(a))  # noqa: E731
        for i in range(self.n_step):
            nxt = o(self.sequence[i][0])
            self.target_critic(nxt, self.target_actor(nxt))
        for i in range(len(self.sequence) - self.n_step):
            obs, action, nxt = o(self.sequence[i][0]), t(self.sequence[i][1]), o(self.sequence[i + self.n_step][0])
            q = self.critic(obs, action).cpu().numpy()
            q_next = self.target_critic(nxt, self.target_actor(nxt)).cpu().numpy()
            if i >= self.burn_in_length:
                terminal = self.sequence[i + self.n_step - 1][3][0]
                if invertible:
                    q_next = inverse_value_rescale(torch.tensor(q_next), eps).numpy()
                y = self.sequence[i][2][0] + (self.gamma ** self.n_step) * (1.0 - terminal) * q_next
                y = (value_rescale(torch.tensor(y), eps) if invertible else invertical_vf(torch.tensor(y))).numpy()
                self.td_loss.append((q - y).mean())
            if i >= self.sequence_length:
                td = np.array(list(self.td_loss), dtype=np.float32)
                self.priority.append(calc_priority(np.abs(td) if opt.priority_metric == "abs" else td ** 2.0))

    def run(self, max_episodes=None):
        episode = step = 0
        while max_episodes is None or episode < max_episodes:
            time_step = self.env.reset()
            obs = get_obs(time_step.observation)
            for _, net in self._nets():
                net.reset_state()
            if self.noise is not None:
                self.noise.reset([0])
            self.sequence, self.recurrent_state, self.priority = [], [], []
            episode += 1
            reward_sum = 0.0
            while not time_step.last():
                states = [net.get_state() for _, net in self._nets()]
                with torch.no_grad():
                    x = self._obs(torch.from_numpy(obs).to(self.device))
                    action = self.actor(x)
                    self.critic(x, action)
                    self.target_critic(x, self.target_actor(x))
                if self.noise is None:
                    action = np.clip(action.cpu().numpy()[0] + np.random.normal(0, 0.3, self.action_size), -1, 1)
                else:
                    action = self.noise.actions(action.cpu().numpy(), step)[0]
                reward = 0.0
                for _ in range(4):                                        # action repeat, actor.py:152-157
                    time_step = self.env.step(action)
                    next_obs = get_obs(time_step.observation)
                    reward += time_step.reward or 0.0
                    if time_step.last():
                        break
                reward_sum += reward
                step += 1
                self.sequence.append((obs[0], action.astype(np.float32), [reward], [1.0 if time_step.last() else 0.0]))
                self.recurrent_state.append([[h[0], c[0]] for h, c in states])
                obs = next_obs.copy()
                if step % self.actor_parameter_update_interval == 0:
                    self.load_model()
            if self.actor_id == 0:
                print('episode:', episode, 'step:', step, 'reward:', reward_sum)
            if self.episode_log is not None:
                metrics.append_csv(self.episode_log, metrics.EPISODE_COLUMNS,
                                   [(self.actor_id, episode, step, len(self.sequence), reward_sum,
                                     len(self.sequence) >= self.sequence_length)])
            if len(self.sequence) >= self.sequence_length:
                pad = (np.zeros(self.obs_size, np.float32), np.zeros(self.action_size, np.float32), [0.0], [1.0])
                self.sequence.extend([(pad[0].copy(), pad[1].copy(), [0.0], [1.0]) for _ in range(self.n_step)])
                self.calc_nstep_reward()
                self.calc_priorities()
                self.memory.add(self.sequence, self.recurrent_state, self.priority)
            if len(self.memory.memory) > self.memory_save_interval:
                self.memory.save(self.actor_id)

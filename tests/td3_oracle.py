"""Float64 restatement of TD3's target for the learner, on top of oracle/learner_oracle.py (unchanged).

- `philox4x32_10` / `normal` / `smooth`: the library's target-noise generator in numpy uint32 arithmetic
  (include/r2d2_b200.h r2d2_target_smoothing): key = (seed, rank), counter = (e >> 2, iter_lo, iter_hi, 0);
  words (x0, x1) serve e % 4 in {0, 1}, (x2, x3) serve {2, 3}; u = (2 (x >> 9) + 1) 2^-24;
  z = sqrt(-2 ln u_a) {cos, sin}(2 pi u_b); a' = clip(mu + clip(sigma z, -c, c), -1, 1).
- `TD3Oracle`: an OracleLearner whose own iteration adds the twin critic (critic 2 and its target from the zero state,
  q' = min(q'_1, q'_2), each critic its own MSE against the same y and its own BPTT, two Adams), target policy smoothing
  keyed on the iteration index, the Polyak update of optim_oracle, gradient-norm clipping (joint over both critics, per
  net otherwise) and any TD function of rescale_oracle (`td=`).  It reuses net_forward, net_backward, adam_step and the TD
  function, in the base iteration's order, so with the twin off and sigma = 0 it returns the base's arrays exactly.
  `iteration(shards)` with several shards models the data-parallel learner: every rank's gradients with its own noise
  key, averaged, one optimiser step.
"""
import numpy as np

from oracle import learner_oracle as lo

_M0, _M1, _W0, _W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
_MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr: four uint32 arrays (or scalars), key: two.  Returns the four output words as uint32 arrays."""
    c = [np.asarray(x, np.uint64) & _MASK for x in ctr]
    k0, k1 = (np.asarray(x, np.uint64) & _MASK for x in key)
    for r in range(10):
        if r:
            k0, k1 = (k0 + np.uint64(_W0)) & _MASK, (k1 + np.uint64(_W1)) & _MASK
        p0 = np.uint64(_M0) * c[0]
        p1 = np.uint64(_M1) * c[2]
        hi0, lo0 = p0 >> np.uint64(32), p0 & _MASK
        hi1, lo1 = p1 >> np.uint64(32), p1 & _MASK
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
    return [x.astype(np.uint32) for x in c]


def unit_open(x):
    return (2.0 * (np.asarray(x, np.uint32) >> np.uint32(9)).astype(np.float64) + 1.0) * 2.0 ** -24


def normal(n, seed, rank, it):
    """z_e for e < n."""
    e = np.arange(n, dtype=np.uint64)
    g = e >> np.uint64(2)
    z = np.zeros_like(g)
    x = philox4x32_10((g, z + np.uint64(it & 0xFFFFFFFF), z + np.uint64(it >> 32), z), (z + np.uint64(seed), z + np.uint64(rank)))
    pair = ((e & np.uint64(3)) >> np.uint64(1)).astype(bool)
    ua = unit_open(np.where(pair, x[2], x[0]))
    ub = unit_open(np.where(pair, x[3], x[1]))
    rad = np.sqrt(-2.0 * np.log(ua))
    odd = (e & np.uint64(1)).astype(bool)
    return rad * np.where(odd, np.sin(2.0 * np.pi * ub), np.cos(2.0 * np.pi * ub))


def smooth(mu, sigma, clip, seed, rank, it):
    mu = np.asarray(mu, np.float64)
    noise = np.clip(sigma * normal(mu.size, seed, rank, it).reshape(mu.shape), -clip, clip)
    return np.clip(mu + noise, -1.0, 1.0)


def _grad_norm(*grads):
    return float(np.sqrt(sum(float(np.sum(np.square(g[k], dtype=np.float64))) for g in grads for k in lo.PARAM_KEYS)))


class TD3Oracle(lo.OracleLearner):
    def __init__(self, actor, critic, target_actor=None, target_critic=None, *, critic2=None, target_critic2=None,
                 twin=False, sigma=0.0, noise_clip=0.5, seed=0, rank=0, target_tau=1.0, grad_clip=0.0, td=None, **kw):
        super().__init__(actor, critic, target_actor, target_critic, **kw)
        cv = lambda d: {k: np.asarray(d[k], dtype=self.dtype).copy() for k in lo.PARAM_KEYS}  # noqa: E731
        self.twin = twin
        if twin:
            self.critic2 = cv(critic2)
            self.target_critic2 = cv(target_critic2 if target_critic2 is not None else critic2)
            self.critic2_adam = {}
        self.sigma, self.noise_clip, self.seed, self.rank = sigma, noise_clip, seed, rank
        self.target_tau, self.grad_clip = target_tau, grad_clip
        self.td = td
        self.norms = {}

    def _td(self, *a, **k):
        return (self.td or lo.td_targets_and_priorities)(*a, **k)

    def _critic_grads(self, batch, it, rank):
        dt = self.dtype
        Bn, L, n = self.burn_in, self.learning, self.n_step
        obs, act = np.asarray(batch["obs"], dt), np.asarray(batch["act"], dt)
        T_all, B, _ = obs.shape
        rew = np.asarray(batch["rew"], dt).reshape(T_all, B)
        term = np.asarray(batch["term"], dt).reshape(T_all, B)
        st = {k: np.asarray(batch[k], dt) for k in ("ta_state", "c_state", "tc_state")}
        ta = lo.net_forward(self.target_actor, obs[:Bn + n + L], st["ta_state"][0], st["ta_state"][1], critic=False)
        act_next = ta["out"][Bn + n:]
        if self.sigma > 0:
            act_next = smooth(act_next, self.sigma, self.noise_clip, self.seed, rank, it)
        tc_in = np.concatenate((obs[:Bn + n + L], np.concatenate((act[:Bn + n], act_next), 0)), 2)
        tc = lo.net_forward(self.target_critic, tc_in, st["tc_state"][0], st["tc_state"][1], critic=True)
        q_next = tc["out"][Bn + n:]
        zeros = np.zeros((B, self.critic["l2.weight_hh"].shape[1]), dt)
        if self.twin:
            q_next = np.minimum(q_next, lo.net_forward(self.target_critic2, tc_in, zeros, zeros, critic=True)["out"][Bn + n:])
        c_in = np.concatenate((obs[:Bn + L], act[:Bn + L]), 2)
        c1 = lo.net_forward(self.critic, c_in, st["c_state"][0], st["c_state"][1], critic=True)
        q = c1["out"][Bn:]
        y, critic_loss, dq, td_sq, prio = self._td(q, q_next, rew, term, burn_in=Bn, learning=L, n_step=n,
                                                   gamma=self.gamma)
        d_out = np.concatenate((np.zeros((Bn,) + dq.shape[1:], dt), dq), 0)
        critic_grad, _, _ = lo.net_backward(self.critic, c1, d_out, critic=True)
        out = {"critic_loss": critic_loss, "priority": prio, "average_td_loss": td_sq.reshape(-1), "q": q, "y": y,
               "act_next": act_next, "q_next": q_next, "grads": {"critic": critic_grad}}
        if self.twin:
            c2 = lo.net_forward(self.critic2, c_in, zeros, zeros, critic=True)
            q2 = c2["out"][Bn:]
            _, loss2, dq2, _, _ = self._td(q2, q_next, rew, term, burn_in=Bn, learning=L, n_step=n, gamma=self.gamma)
            d_out2 = np.concatenate((np.zeros((Bn,) + dq2.shape[1:], dt), dq2), 0)
            out["grads"]["critic2"], _, _ = lo.net_backward(self.critic2, c2, d_out2, critic=True)
            out.update(q2=q2, critic2_loss=loss2)
        return out

    def _actor_grads(self, batch):
        dt = self.dtype
        Bn, L = self.burn_in, self.learning
        obs = np.asarray(batch["obs"], dt)
        B = obs.shape[1]
        zeros = np.zeros((B, self.actor["l2.weight_hh"].shape[1]), dt)
        a1 = lo.net_forward(self.actor, obs[Bn:Bn + L], zeros, zeros, critic=False, repeat=2)
        mu = a1["out"][1::2]
        c2 = lo.net_forward(self.critic, np.concatenate((obs[Bn:Bn + L], mu), 2), zeros, zeros, critic=True)
        q_pi = c2["out"]
        actor_loss = float(np.mean(-q_pi))
        dq_pi = np.full(q_pi.shape, -1.0 / q_pi.size, dt)
        _, dx, _ = lo.net_backward(self.critic, c2, dq_pi, critic=True, want_wgrad=False, want_dx=True)
        d_out_a = np.zeros_like(a1["out"])
        d_out_a[1::2] = dx[:, :, obs.shape[2]:]
        actor_grad, _, _ = lo.net_backward(self.actor, a1, d_out_a, critic=False)
        return actor_grad, actor_loss

    @staticmethod
    def _mean(gs):
        if len(gs) == 1:
            return gs[0]
        return {k: sum(g[k] for g in gs) / len(gs) for k in lo.PARAM_KEYS}

    def _clip(self, *grads):
        n = _grad_norm(*grads)
        if self.grad_clip > 0:
            c = min(1.0, self.grad_clip / (n + 1e-6))
            for g in grads:
                for k in lo.PARAM_KEYS:
                    g[k] *= c
        return n

    def iteration(self, batch, keep=True, grad_hook=None):
        """batch: one batch, or a list of rank shards (rank r draws noise with key (seed, r))."""
        shards = batch if isinstance(batch, (list, tuple)) else [batch]
        ranks = [self.rank] if len(shards) == 1 else list(range(len(shards)))
        it = self.step_count
        self.step_count += 1
        outs = [self._critic_grads(b, it, r) for b, r in zip(shards, ranks)]
        cg = self._mean([o["grads"]["critic"] for o in outs])
        if grad_hook is not None:
            grad_hook("critic", cg)
        nets = [(self.critic, cg, self.critic_adam)]
        if self.twin:
            cg2 = self._mean([o["grads"]["critic2"] for o in outs])
            if grad_hook is not None:
                grad_hook("critic2", cg2)
            nets.append((self.critic2, cg2, self.critic2_adam))
        if self.grad_clip > 0:
            self.norms["critic"] = self._clip(*[g for _, g, _ in nets])
        for p, g, st in nets:
            lo.adam_step(p, g, st, self.critic_lr)
        ag = [self._actor_grads(b) for b in shards]
        actor_grad = self._mean([a for a, _ in ag])
        if grad_hook is not None:
            grad_hook("actor", actor_grad)
        if self.grad_clip > 0:
            self.norms["actor"] = self._clip(actor_grad)
        lo.adam_step(self.actor, actor_grad, self.actor_adam, self.actor_lr)
        if self.step_count % self.target_interval == 0:
            t = self.target_tau
            pairs = [("target_actor", self.actor), ("target_critic", self.critic)]
            if self.twin:
                pairs.append(("target_critic2", self.critic2))
            for name, net in pairs:
                if t == 1.0:
                    setattr(self, name, {k: v.copy() for k, v in net.items()})
                else:
                    old = getattr(self, name)
                    setattr(self, name, {k: old[k] * (1.0 - t) + net[k] * t for k in lo.PARAM_KEYS})
        o = outs[0]
        res = {"critic_loss": o["critic_loss"], "actor_loss": ag[0][1], "priority": o["priority"],
               "average_td_loss": o["average_td_loss"]}
        if keep:
            A = o["q"].shape[2]
            res.update(q_value=o["q"].reshape(-1, A), target_q_value=o["y"].reshape(-1, A), critic_grad=cg,
                       actor_grad=actor_grad, act_next=o["act_next"], q_next=o["q_next"])
            if self.twin:
                res.update(q_value2=o["q2"].reshape(-1, A), critic2_loss=o["critic2_loss"])
            res["shards"] = outs
        return res

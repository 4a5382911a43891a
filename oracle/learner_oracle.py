"""numpy restatement (float64 by default) of the learner hot path, written as the SAME
decomposition the CUDA library uses: hoisted input GEMMs -> serial LSTM scan -> head, manual BPTT.

TEST INFRASTRUCTURE: only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may
import this; the product path never does.  Pure numpy, no autograd: every gradient formula that
the CUDA kernels implement is spelled out here and pinned against the real reference's autograd
through tests/golden/*.npz (tests/test_oracle_golden.py).

Reference lines restated
  net forward            models.py:32-40 (actor), :74-83 (critic; tanh at :81 discarded, A outputs)
  LSTMCell gate order    torch.nn.LSTMCell: i, f, g, o; b_ih + b_hh  (used at models.py:37,80)
  burn-in / unroll       learner.py:92-109  (dead actor burn-in learner.py:92 is skipped: its state
                         is dropped at learner.py:117 before any use, quirk Q5)
  n-step target          learner.py:107-108, utils.py:20-21 (h without h^-1, rewards pre-summed)
  critic loss / Adam     learner.py:111-114 (MSE mean over L*B*A; grads flow through burn-in, Q4)
  actor update           learner.py:117-128 (zero state, actor cell stepped twice per row, post-step
                         critic, loss = mean(-Q))
  priorities             learner.py:135-138, utils.py:17-18 (slice [b:-1:B], quirk Q10)
  hard target update     learner.py:63-65,131-132

Every learner option the library has beyond the reference is a keyword of `OracleLearner` named as in `PathConfig`, and
its default is the reference's behaviour, computed with the same float64 operations in the same order:
  importance weights     batch["is_weight"] [B]: loss sum_b w_b sum (q - y)^2 / (L*B*A); td_sq and priorities unweighted
  value_rescaling        "invertible": y = h_eps(R + gamma^n (1-d) h_eps^-1(Q')), eps = rescaling_eps
  priority_metric        "abs": priorities over sqrt(td_sq) instead of td_sq
  target_tau             on target-update iterations target <- target (1 - tau) + tau param' (utils.soft_update)
  grad_clip              g <- g min(1, M / (N + 1e-6)), N the L2 norm of the net's whole gradient block (joint over both
                         critics with the twin), as torch.nn.utils.clip_grad_norm_
  twin                   TD3's twin critic: critic 2 and its target from the zero state, q' = min(q'_1, q'_2), each critic
                         its own loss against the same y and its own BPTT, one Adam and one clip over both
  target_noise           TD3's target policy smoothing (oracle/target_noise.py), keyed on (seed, rank) and the iteration
`iteration` also takes a list of rank shards: every rank's gradients with its own noise key, averaged, one optimiser
step - the data-parallel learner.
"""
from __future__ import annotations

import numpy as np

from oracle.target_noise import smooth

PARAM_KEYS = ("l1.weight", "l1.bias", "l2.weight_ih", "l2.weight_hh", "l2.bias_ih", "l2.bias_hh",
              "l3.weight", "l3.bias")


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def value_rescale(x):
    return np.sign(x) * (np.sqrt(np.abs(x) + 1.0) - 1.0)


def h_eps(x, eps):
    """h_eps(x) = sign(x)(sqrt(|x|+1) - 1) + eps x in the library's form that does not cancel near 0."""
    x = np.asarray(x, np.float64)
    a = np.abs(x)
    return np.sign(x) * (a / (np.sqrt(a + 1.0) + 1.0)) + eps * x


def h_eps_inv(x, eps):
    """h_eps^-1(x) = sign(x) v (v+2) with v = 2|x| / ((1+2eps) + sqrt((1+2eps)^2 + 4 eps |x|))."""
    x = np.asarray(x, np.float64)
    a = np.abs(x)
    c = 1.0 + 2.0 * eps
    v = 2.0 * a / (c + np.sqrt(c * c + 4.0 * eps * a))
    return np.sign(x) * (v * (v + 2.0))


def n_step_target(r, cont, q_next, rescaling="reference", eps=1e-3):
    """y from the n-step reward sum r, cont = gamma^n (1 - d) and the bootstrap q_next."""
    if rescaling == "invertible":
        return h_eps(r + cont * h_eps_inv(q_next, eps), eps)
    return value_rescale(r + cont * q_next)


def net_forward(p, x, h0, c0, *, critic: bool, repeat: int = 1):
    """x [T,B,I] -> saved activations.  steps = T*repeat; step s consumes row s//repeat.
    Saved: z1 [T,B,H]; gates [S,B,4H] post-activation (i,f,g,o); hs, cs [S+1,B,H] (slot 0 = initial
    state); out [S,B,A]."""
    T, B, _ = x.shape
    H = p["l2.weight_hh"].shape[1]
    z1 = np.tanh(x @ p["l1.weight"].T + p["l1.bias"])
    gin = z1 @ p["l2.weight_ih"].T + (p["l2.bias_ih"] + p["l2.bias_hh"])
    S = T * repeat
    hs = np.zeros((S + 1, B, H), x.dtype)
    cs = np.zeros((S + 1, B, H), x.dtype)
    gates = np.zeros((S, B, 4 * H), x.dtype)
    hs[0], cs[0] = h0, c0
    whh_t = p["l2.weight_hh"].T
    for s in range(S):
        g = gin[s // repeat] + hs[s] @ whh_t
        i, f, gg, o = (_sigmoid(g[:, :H]), _sigmoid(g[:, H:2 * H]), np.tanh(g[:, 2 * H:3 * H]),
                       _sigmoid(g[:, 3 * H:]))
        cs[s + 1] = f * cs[s] + i * gg
        hs[s + 1] = o * np.tanh(cs[s + 1])
        gates[s] = np.concatenate((i, f, gg, o), 1)
    if critic:
        out = hs[1:] @ p["l3.weight"].T + p["l3.bias"]
    else:
        out = np.tanh(np.tanh(hs[1:]) @ p["l3.weight"].T + p["l3.bias"])
    return {"x": x, "z1": z1, "gates": gates, "hs": hs, "cs": cs, "out": out, "repeat": repeat}


def lstm_scan(gin, whh, h0=None, c0=None, dh_head=None, *, repeat=1, head_first_step=0):
    """The recurrence alone, as r2d2_lstm_scan_forward / _backward compute it: gates_s = gin[s // repeat] + h_{s-1}
    W_hh^T for s < S = T * repeat (h0 / c0 None: zero state).  Step s >= head_first_step with (s - head_first_step) %
    repeat == repeat - 1 adds dh_head row (s - head_first_step) // repeat to dL/dh_s (dh_head None: forward only).
    Returns hs, cs [S+1,B,H] (slot 0 = initial state), gates [S,B,4H] post-activation (i, f, g, o), head_in [T,B,H] =
    tanh(h) after the last step of each row and, with dh_head, dgates [S,B,4H] and dgin [T,B,4H] (dgates summed per
    input row)."""
    T, B, H4 = gin.shape
    H, S = H4 // 4, T * repeat
    hs, cs = np.zeros((S + 1, B, H)), np.zeros((S + 1, B, H))
    gates = np.empty((S, B, H4))
    if h0 is not None:
        hs[0] = h0
    if c0 is not None:
        cs[0] = c0
    for s in range(S):
        pre = gin[s // repeat] + hs[s] @ whh.T
        i, f, g, o = _sigmoid(pre[:, :H]), _sigmoid(pre[:, H:2 * H]), np.tanh(pre[:, 2 * H:3 * H]), _sigmoid(pre[:, 3 * H:])
        cs[s + 1] = f * cs[s] + i * g
        hs[s + 1] = o * np.tanh(cs[s + 1])
        gates[s] = np.concatenate((i, f, g, o), 1)
    out = {"hs": hs, "cs": cs, "gates": gates, "head_in": np.tanh(hs[repeat::repeat])}
    if dh_head is None:
        return out
    dgates, dgin = np.empty_like(gates), np.zeros_like(gin)
    dh_rec, dc_next = np.zeros((B, H)), np.zeros((B, H))
    for s in range(S - 1, -1, -1):
        i, f, g, o = gates[s, :, :H], gates[s, :, H:2 * H], gates[s, :, 2 * H:3 * H], gates[s, :, 3 * H:]
        rel = s - head_first_step
        dh = dh_rec + (dh_head[rel // repeat] if rel >= 0 and rel % repeat == repeat - 1 else 0.0)
        tc = np.tanh(cs[s + 1])
        dc = dc_next + dh * o * (1 - tc * tc)
        dgates[s] = np.concatenate((dc * g * i * (1 - i), dc * cs[s] * f * (1 - f), dc * i * (1 - g * g),
                                    dh * tc * o * (1 - o)), 1)
        dc_next = dc * f
        dh_rec = dgates[s] @ whh
        dgin[s // repeat] += dgates[s]
    out.update(dgates=dgates, dgin=dgin)
    return out


def net_backward(p, sv, d_out, *, critic: bool, want_wgrad: bool = True, want_dx: bool = False):
    """Manual BPTT.  d_out [S,B,A] (zero rows where the output is unused)."""
    x, z1, gates, hs, cs, out, repeat = (sv[k] for k in ("x", "z1", "gates", "hs", "cs", "out", "repeat"))
    S, B, _ = d_out.shape
    T = S // repeat
    H = hs.shape[2]
    g = {}
    if critic:
        d_pre = d_out
        head_in = hs[1:]
        d_h_head = d_pre @ p["l3.weight"]
    else:
        d_pre = d_out * (1.0 - out * out)
        head_in = np.tanh(hs[1:])
        d_h_head = (d_pre @ p["l3.weight"]) * (1.0 - head_in * head_in)
    if want_wgrad:
        g["l3.weight"] = np.einsum("sba,sbh->ah", d_pre, head_in)
        g["l3.bias"] = d_pre.sum((0, 1))
    d_gates = np.zeros_like(gates)
    dh_rec = np.zeros((B, H), x.dtype)
    dc_next = np.zeros((B, H), x.dtype)
    whh = p["l2.weight_hh"]
    for s in range(S - 1, -1, -1):
        i, f, gg, o = (gates[s][:, :H], gates[s][:, H:2 * H], gates[s][:, 2 * H:3 * H], gates[s][:, 3 * H:])
        tc = np.tanh(cs[s + 1])
        dh = d_h_head[s] + dh_rec
        d_o = dh * tc * o * (1.0 - o)
        dc = dc_next + dh * o * (1.0 - tc * tc)
        d_i = dc * gg * i * (1.0 - i)
        d_f = dc * cs[s] * f * (1.0 - f)
        d_g = dc * i * (1.0 - gg * gg)
        dc_next = dc * f
        d_gates[s] = np.concatenate((d_i, d_f, d_g, d_o), 1)
        dh_rec = d_gates[s] @ whh
    d_gin = d_gates.reshape(T, repeat, B, 4 * H).sum(1)
    if want_wgrad:
        g["l2.weight_hh"] = np.einsum("sbg,sbh->gh", d_gates, hs[:-1])
        g["l2.weight_ih"] = np.einsum("tbg,tbh->gh", d_gin, z1)
        g["l2.bias_ih"] = d_gin.sum((0, 1))
        g["l2.bias_hh"] = g["l2.bias_ih"].copy()
    d_p1 = (d_gin @ p["l2.weight_ih"]) * (1.0 - z1 * z1)
    if want_wgrad:
        g["l1.weight"] = np.einsum("tbh,tbi->hi", d_p1, x)
        g["l1.bias"] = d_p1.sum((0, 1))
    dx = d_p1 @ p["l1.weight"] if want_dx else None
    return g, dx, {"d_gates": d_gates, "d_h_head": d_h_head, "d_p1": d_p1, "dh0": dh_rec, "dc0": dc_next}


def adam_step(p, g, state, lr, b1=0.9, b2=0.999, eps=1e-8):
    """torch.optim.Adam defaults (learner.py:50,52): no weight decay, no amsgrad."""
    state["t"] = state.get("t", 0) + 1
    t = state["t"]
    for k in PARAM_KEYS:
        m = state.setdefault("m/" + k, np.zeros_like(p[k]))
        v = state.setdefault("v/" + k, np.zeros_like(p[k]))
        m *= b1
        m += (1 - b1) * g[k]
        v *= b2
        v += (1 - b2) * g[k] * g[k]
        denom = np.sqrt(v) / np.sqrt(1 - b2 ** t) + eps
        p[k] = p[k] - (lr / (1 - b1 ** t)) * (m / denom)


def weighted_loss(diff, is_weight):
    """The importance-weighted critic loss sum_b w_b sum_{i,a} diff^2 / (L*B*A) and its gradient 2 w_b diff / (L*B*A)."""
    w = np.asarray(is_weight, diff.dtype).reshape(1, -1, 1)
    return float(np.sum(w * diff * diff) / diff.size), 2.0 * w * diff / diff.size


def td_targets_and_priorities(q, q_next, rew, term, *, burn_in, learning, n_step, gamma, eta=0.9,
                              rescaling="reference", eps=1e-3, metric="squared", is_weight=None):
    """q, q_next [L,B,A]; rew, term [T',B]; is_weight [B] or None.  Returns target y [L,B,A], loss, dq, td_sq [L,B],
    priority [B]."""
    L, B, A = q.shape
    r = rew[burn_in:burn_in + learning][:, :, None]
    d = term[burn_in + n_step - 1:burn_in + n_step - 1 + learning][:, :, None]
    y = n_step_target(r, gamma ** n_step * (1.0 - d), q_next, rescaling, eps)
    diff = q - y
    if is_weight is None:
        loss = float(np.mean(diff * diff))
        dq = 2.0 * diff / diff.size
    else:
        loss, dq = weighted_loss(diff, is_weight)
    td_sq = np.mean(diff * diff, axis=2)                      # [L,B]
    flat = (np.sqrt(td_sq) if metric == "abs" else td_sq).reshape(-1)   # index i*B + b (time-major blocks of B)
    prio = np.zeros(B, q.dtype)
    for b in range(B):
        series = flat[b:-1:B]                                 # learner.py:137; drops the very last element
        prio[b] = eta * series.max() + (1.0 - eta) * series.mean()
    return y, loss, dq, td_sq, prio


def grad_norm(*grads):
    """L2 norm over every parameter of the given gradient dicts, in float64."""
    return float(np.sqrt(sum(float(np.sum(np.square(g[k], dtype=np.float64))) for g in grads for k in PARAM_KEYS)))


def _mean(gs):
    if len(gs) == 1:
        return gs[0]
    return {k: sum(g[k] for g in gs) / len(gs) for k in PARAM_KEYS}


class OracleLearner:
    """State (params, targets, Adam moments, step counter) + one iteration of the necessary work."""

    def __init__(self, actor, critic, target_actor=None, target_critic=None, *, burn_in=20, learning=40,
                 n_step=5, gamma=0.997, actor_lr=1e-4, critic_lr=1e-3, target_interval=500, target_tau=1.0,
                 grad_clip=0.0, value_rescaling="reference", rescaling_eps=1e-3, priority_metric="squared",
                 twin=False, critic2=None, target_critic2=None, target_noise=0.0, target_noise_clip=0.5,
                 target_noise_seed=0, rank=0, dtype=np.float64):
        cv = lambda d: {k: np.asarray(d[k], dtype=dtype).copy() for k in PARAM_KEYS}  # noqa: E731
        self.actor, self.critic = cv(actor), cv(critic)
        self.target_actor = cv(target_actor if target_actor is not None else actor)
        self.target_critic = cv(target_critic if target_critic is not None else critic)
        self.twin = twin
        if twin:
            self.critic2 = cv(critic2)
            self.target_critic2 = cv(target_critic2 if target_critic2 is not None else critic2)
        self.burn_in, self.learning, self.n_step, self.gamma = burn_in, learning, n_step, gamma
        self.actor_lr, self.critic_lr, self.target_interval = actor_lr, critic_lr, target_interval
        self.target_tau, self.grad_clip = target_tau, grad_clip
        # The TD function gets only the options that differ from the reference's, and the importance weights are applied
        # to its target here, so OracleLearner calls it with the reference's arguments unless an option is on.
        self.td_options = {k: v for k, v, ref in (("rescaling", value_rescaling, "reference"), ("eps", rescaling_eps, 1e-3),
                                                  ("metric", priority_metric, "squared")) if v != ref}
        self.target_noise, self.target_noise_clip = target_noise, target_noise_clip
        self.target_noise_seed, self.rank = target_noise_seed, rank
        self.dtype = dtype
        self.actor_adam, self.critic_adam, self.critic2_adam = {}, {}, {}
        self.norms = {}                                       # pre-clip gradient norms of the last iteration
        self.step_count = 0

    def _critic_pass(self, batch, it, rank):
        """One shard's targets, TD and critic gradients (learner.py:92-114)."""
        dt = self.dtype
        Bn, L, n = self.burn_in, self.learning, self.n_step
        obs, act = np.asarray(batch["obs"], dt), np.asarray(batch["act"], dt)
        T_all, B, _ = obs.shape
        rew = np.asarray(batch["rew"], dt).reshape(T_all, B)
        term = np.asarray(batch["term"], dt).reshape(T_all, B)
        st = {k: np.asarray(batch[k], dt) for k in ("ta_state", "c_state", "tc_state")}
        w = batch.get("is_weight")
        w = None if w is None else np.asarray(w, dt)
        # --- target actor over rows [0, Bn+n+L) (learner.py:94,106)
        ta = net_forward(self.target_actor, obs[:Bn + n + L], st["ta_state"][0], st["ta_state"][1], critic=False)
        act_next = ta["out"][Bn + n:]
        if self.target_noise > 0:
            act_next = smooth(act_next, self.target_noise, self.target_noise_clip, self.target_noise_seed, rank, it)
        # --- target critic: stored actions for burn-in rows, target-actor actions after (learner.py:95,106)
        tc_in = np.concatenate((obs[:Bn + n + L], np.concatenate((act[:Bn + n], act_next), 0)), 2)
        tc = net_forward(self.target_critic, tc_in, st["tc_state"][0], st["tc_state"][1], critic=True)
        q_next = tc["out"][Bn + n:]
        zeros = np.zeros((B, self.critic["l2.weight_hh"].shape[1]), dt)
        if self.twin:
            q_next = np.minimum(q_next, net_forward(self.target_critic2, tc_in, zeros, zeros, critic=True)["out"][Bn + n:])
        # --- online critic over rows [0, Bn+L) with stored actions (learner.py:93,105)
        c_in = np.concatenate((obs[:Bn + L], act[:Bn + L]), 2)
        out = {"act_next": act_next, "q_next": q_next, "grads": {}}
        for name, h0 in (("critic", st["c_state"]), ("critic2", (zeros, zeros)))[:1 + self.twin]:
            net = getattr(self, name)
            sv = net_forward(net, c_in, h0[0], h0[1], critic=True)
            q = sv["out"][Bn:]
            y, loss, dq, td_sq, prio = td_targets_and_priorities(
                q, q_next, rew, term, burn_in=Bn, learning=L, n_step=n, gamma=self.gamma, **self.td_options)
            if w is not None:
                loss, dq = weighted_loss(q - y, w)
            d_out = np.concatenate((np.zeros((Bn,) + dq.shape[1:], dt), dq), 0)
            out["grads"][name], _, _ = net_backward(net, sv, d_out, critic=True)
            if name == "critic":
                out.update(q=q, y=y, critic_loss=loss, td_sq=td_sq, priority=prio)
            else:
                out.update(q2=q, critic2_loss=loss)
        return out

    def _actor_pass(self, batch):
        """One shard's actor loss and gradient through the post-step critic (learner.py:117-128)."""
        dt = self.dtype
        Bn, L = self.burn_in, self.learning
        obs = np.asarray(batch["obs"], dt)
        B = obs.shape[1]
        zeros = np.zeros((B, self.actor["l2.weight_hh"].shape[1]), dt)
        a1 = net_forward(self.actor, obs[Bn:Bn + L], zeros, zeros, critic=False, repeat=2)
        mu = a1["out"][1::2]                                          # output of the second call per row
        c2 = net_forward(self.critic, np.concatenate((obs[Bn:Bn + L], mu), 2), zeros, zeros, critic=True)
        q_pi = c2["out"]
        dq_pi = np.full(q_pi.shape, -1.0 / q_pi.size, dt)
        _, dx, _ = net_backward(self.critic, c2, dq_pi, critic=True, want_wgrad=False, want_dx=True)
        d_mu = dx[:, :, obs.shape[2]:]
        d_out_a = np.zeros_like(a1["out"])
        d_out_a[1::2] = d_mu
        grad, _, _ = net_backward(self.actor, a1, d_out_a, critic=False)
        return {"grad": grad, "loss": float(np.mean(-q_pi)), "mu": mu, "q_pi": q_pi, "d_mu": d_mu}

    def _optimise(self, names, grads, lr, grad_hook, pre_clip):
        """grad_hook, then one clip over the nets' joint gradient block, then each net's Adam step."""
        for name in names:
            if grad_hook is not None:
                grad_hook(name, grads[name])
            pre_clip[name] = {k: v.copy() for k, v in grads[name].items()}
        norm = self.norms[names[0]] = grad_norm(*(grads[name] for name in names))
        if self.grad_clip > 0:
            c = min(1.0, self.grad_clip / (norm + 1e-6))
            for name in names:
                for k in PARAM_KEYS:
                    grads[name][k] *= c
        for name in names:
            adam_step(getattr(self, name), grads[name], getattr(self, name + "_adam"), lr)

    def iteration(self, batch, keep=True, grad_hook=None):
        """batch: one batch, or a list of rank shards (rank r draws its noise with key (seed, r)).  grad_hook(net_name,
        grads_dict) may replace the (shard-averaged) gradients in place before clipping and the optimiser step (used to
        model the data-parallel all-reduce: mean of per-rank gradients == gradient of the global batch)."""
        shards = batch if isinstance(batch, (list, tuple)) else [batch]
        ranks = [self.rank] if len(shards) == 1 else range(len(shards))
        it = self.step_count
        self.step_count += 1
        outs = [self._critic_pass(b, it, r) for b, r in zip(shards, ranks)]
        critics = ("critic", "critic2")[:1 + self.twin]
        grads = {name: _mean([o["grads"][name] for o in outs]) for name in critics}
        pre_clip = {}
        self._optimise(critics, grads, self.critic_lr, grad_hook, pre_clip)
        acts = [self._actor_pass(b) for b in shards]
        grads["actor"] = _mean([a["grad"] for a in acts])
        self._optimise(("actor",), grads, self.actor_lr, grad_hook, pre_clip)
        if self.step_count % self.target_interval == 0:
            t = self.target_tau
            for name in ("actor",) + critics:
                net, old = getattr(self, name), getattr(self, "target_" + name)
                setattr(self, "target_" + name, {k: v.copy() for k, v in net.items()} if t == 1.0 else
                        {k: old[k] * (1.0 - t) + net[k] * t for k in PARAM_KEYS})
        o, a = outs[0], acts[0]
        out = {"critic_loss": o["critic_loss"], "actor_loss": a["loss"], "priority": o["priority"],
               "average_td_loss": o["td_sq"].reshape(-1)}
        if keep:
            A = o["q"].shape[2]
            out.update(q_value=o["q"].reshape(-1, A), target_q_value=o["y"].reshape(-1, A), critic_grad=grads["critic"],
                       actor_grad=grads["actor"], pre_clip_grad=pre_clip,
                       critic_after={k: v.copy() for k, v in self.critic.items()},
                       actor_after={k: v.copy() for k, v in self.actor.items()}, mu=a["mu"], q_pi=a["q_pi"],
                       act_next=o["act_next"], q_next=o["q_next"], d_mu=a["d_mu"])
            if self.twin:
                out.update(q_value2=o["q2"].reshape(-1, A), critic2_loss=o["critic2_loss"])
        return out

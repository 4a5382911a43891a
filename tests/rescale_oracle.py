"""Float64 restatement of R2D2's n-step target options, on top of oracle/learner_oracle.py and oracle/actor_oracle.py
(both unchanged).

- `h(x, eps)` / `h_inv(x, eps)`: h_eps(x) = sign(x)(sqrt(|x|+1) - 1) + eps x and its inverse, in the forms that do not
  cancel near 0 (the library's): h_eps(x) = sign(x) |x| / (sqrt(|x|+1) + 1) + eps x, h_eps^-1(x) = sign(x) v (v+2) with
  v = 2|x| / ((1+2eps) + sqrt((1+2eps)^2 + 4 eps |x|)).
- `td(rescaling, eps, metric, is_weight)`: a drop-in for learner_oracle.td_targets_and_priorities.  "invertible": the
  target is h_eps(R + gamma^n (1-d) h_eps^-1(Q')); "abs": the priority is eta max + (1-eta) mean over the [b:-1:B] slice of
  m = sqrt(td_sq) instead of td_sq.  The loss (MSE, weighted by is_weight when given), dq and td_sq keep their meaning.
- `iteration(learner, batch, ...)` runs OracleLearner.iteration (or a subclass's, e.g. optim_oracle.PolyakOracle) with it.
- `episode_priorities(...)`: the actor side, actor_oracle.episode_priorities with the same options ("abs": |td| in place
  of td^2, td the mean difference over actions).
"""
import numpy as np

from oracle import actor_oracle
from oracle import learner_oracle as lo

_TD = lo.td_targets_and_priorities


def h(x, eps):
    x = np.asarray(x, np.float64)
    a = np.abs(x)
    return np.sign(x) * (a / (np.sqrt(a + 1.0) + 1.0)) + eps * x


def h_inv(x, eps):
    x = np.asarray(x, np.float64)
    a = np.abs(x)
    c = 1.0 + 2.0 * eps
    v = 2.0 * a / (c + np.sqrt(c * c + 4.0 * eps * a))
    return np.sign(x) * (v * (v + 2.0))


def target(r, cont, q_next, rescaling, eps):
    if rescaling == "invertible":
        return h(r + cont * h_inv(q_next, eps), eps)
    return lo.value_rescale(r + cont * q_next)


def td(rescaling="reference", eps=1e-3, metric="squared", is_weight=None):
    def fn(q, q_next, rew, term, *, burn_in, learning, n_step, gamma, eta=0.9):
        L, B, A = q.shape
        r = rew[burn_in:burn_in + learning][:, :, None]
        d = term[burn_in + n_step - 1:burn_in + n_step - 1 + learning][:, :, None]
        y = target(r, gamma ** n_step * (1.0 - d), q_next, rescaling, eps)
        diff = q - y
        w = np.ones((1, B, 1)) if is_weight is None else np.asarray(is_weight, np.float64).reshape(1, -1, 1)
        loss = float(np.sum(w * diff * diff) / diff.size)
        dq = 2.0 * w * diff / diff.size
        td_sq = np.mean(diff * diff, axis=2)
        flat = (np.sqrt(td_sq) if metric == "abs" else td_sq).reshape(-1)
        prio = np.zeros(B, q.dtype)
        for b in range(B):
            series = flat[b:-1:B]                                 # learner.py:137; drops the very last element
            prio[b] = eta * series.max() + (1.0 - eta) * series.mean()
        return y, loss, dq, td_sq, prio
    return fn


def iteration(learner, batch, rescaling="reference", eps=1e-3, metric="squared", is_weight=None, **kw):
    lo.td_targets_and_priorities = td(rescaling, eps, metric, is_weight)
    try:
        return learner.iteration(batch, **kw)
    finally:
        lo.td_targets_and_priorities = _TD


def episode_priorities(critic, target_actor, target_critic, obs, act, rew, term, *, burn_in, learning, n_step, gamma,
                       eta=0.9, rescaling="reference", eps=1e-3, metric="squared"):
    """obs [N,O], act [N,A], rew [N] (n-step sums), term [N]; N = E + n_step.  Returns priorities [E - burn_in - learning]."""
    if rescaling == "reference" and metric == "squared":
        return actor_oracle.episode_priorities(critic, target_actor, target_critic, obs, act, rew, term, burn_in=burn_in,
                                               learning=learning, n_step=n_step, gamma=gamma, eta=eta)
    f = lambda a: np.asarray(a, np.float32).astype(np.float64)  # noqa: E731
    P = lambda sd: {k: f(v) for k, v in sd.items()}  # noqa: E731
    N = obs.shape[0]
    E = N - n_step
    z = np.zeros((1, np.asarray(critic["l2.weight_hh"]).shape[1]))
    q = lo.net_forward(P(critic), np.concatenate((f(obs[:E]), f(act[:E])), 1)[:, None, :], z, z, critic=True)["out"][:, 0]
    a_t = lo.net_forward(P(target_actor), f(obs)[:, None, :], z, z, critic=False)["out"]
    q_t = lo.net_forward(P(target_critic), np.concatenate((f(obs)[:, None, :], a_t), 2), z, z, critic=True)["out"][:, 0]
    return window_priorities(q, q_t, rew, term, burn_in=burn_in, learning=learning, n_step=n_step, gamma=gamma, eta=eta,
                             rescaling=rescaling, eps=eps, metric=metric)


def window_priorities(q, q_t, rew, term, *, burn_in, learning, n_step, gamma, eta=0.9, rescaling="reference", eps=1e-3,
                      metric="squared"):
    """The windowed part of the actor side on given critic outputs: q [E,A] online, q_t [N,A] target; rew, term [N]."""
    E = q.shape[0]
    tdv = np.zeros(E)
    for i in range(burn_in, E):
        y = target(rew[i], gamma ** n_step * (1.0 - term[i + n_step - 1]), q_t[i + n_step], rescaling, eps)
        tdv[i] = (q[i] - y).mean()
    out = []
    for i in range(burn_in + learning, E):
        w = tdv[i - learning + 1:i + 1]
        w = np.abs(w) if metric == "abs" else w ** 2
        out.append(eta * w.max() + (1 - eta) * w.mean())
    return np.asarray(out, np.float64)

"""TEST INFRASTRUCTURE (checker only; never imported by the product path).

numpy float64 restatement of the actor-side n-step reward pre-sum and initial priorities
(reference actor.py:74-76 `calc_nstep_reward`, :78-107 `calc_priorities`), pinned against
tests/golden/ref_actor_prio.npz (produced by the UNMODIFIED reference, oracle/make_golden.py).

What the reference does, per finished episode of E real rows + n pad rows (actor.py:173):
  * R_i = sum_{j<n} gamma^j r_{i+j} for i < E, computed in place in increasing i (later rows are still raw);
  * all nets restart from the zero state; the target nets first consume rows 0..n-1 (actor.py:86-89), then the loop
    i = 0..E-1 feeds row i to the online critic (stored action) and row i+n to target actor -> target critic:
    every net sees rows 0, 1, 2, ... exactly once;
  * for i >= burn_in: td_i = mean_A( q_i - h(R_i + gamma^n (1 - term_{i+n-1}) q'_{i+n}) )   [mean of the DIFFERENCE];
    a deque of the last `learning` td values; for i >= burn_in + learning the priority
    0.9 max + 0.1 mean of td^2 over the deque, i.e. priority k covers steps k+burn_in+1 .. k+burn_in+learning
    (one step later than the window the learner trains on - the reference's off-by-one, kept).

And the actor's policy step in float64 (reference actor.py `Actor.run`: actor, target actor, critic on the actor's mu,
target critic on the target actor's mu, each net one step from its own recurrent state), with the four-net weights the
policy-step tests draw.
"""
import numpy as np

from oracle import learner_oracle as lo

NETS = ("actor", "target_actor", "critic", "target_critic")


def nstep_rewards(raw, n_step, gamma):
    raw = np.asarray(raw, np.float64)
    out = raw.copy()
    for i in range(len(raw) - n_step):
        out[i] = sum(raw[i + j] * gamma ** j for j in range(n_step))
    return out


def episode_priorities(critic, target_actor, target_critic, obs, act, rew, term, *, burn_in, learning, n_step,
                       gamma, eta=0.9, rescaling="reference", eps=1e-3, metric="squared"):
    """obs [N,O], act [N,A], rew [N] (already n-step sums), term [N]; N = E + n_step.  Returns priorities [E - burn_in - learning].
    rescaling / eps / metric: the TD options of learner_oracle.td_targets_and_priorities."""
    f = lambda a: np.asarray(a, np.float32).astype(np.float64)  # noqa: E731
    N = obs.shape[0]
    E = N - n_step
    H = np.asarray(critic["l2.weight_hh"]).shape[1]
    P = lambda sd: {k: f(v) for k, v in sd.items()}  # noqa: E731
    z = np.zeros((1, H))
    x_c = np.concatenate((f(obs[:E]), f(act[:E])), 1)[:, None, :]
    q = lo.net_forward(P(critic), x_c, z, z, critic=True)["out"][:, 0]                     # [E, A]
    a_t = lo.net_forward(P(target_actor), f(obs)[:, None, :], z, z, critic=False)["out"]    # [N, 1, A]
    x_t = np.concatenate((f(obs)[:, None, :], a_t), 2)
    q_t = lo.net_forward(P(target_critic), x_t, z, z, critic=True)["out"][:, 0]             # [N, A]
    return window_priorities(q, q_t, rew, term, burn_in=burn_in, learning=learning, n_step=n_step, gamma=gamma, eta=eta,
                             rescaling=rescaling, eps=eps, metric=metric)


def window_priorities(q, q_t, rew, term, *, burn_in, learning, n_step, gamma, eta=0.9, rescaling="reference", eps=1e-3,
                      metric="squared"):
    """The windowed part on given critic outputs: q [E,A] online, q_t [N,A] target; rew, term [N].  "abs" takes |td| in
    place of td^2."""
    E = q.shape[0]
    td = np.zeros(E)
    for i in range(burn_in, E):
        y = lo.n_step_target(rew[i], gamma ** n_step * (1.0 - term[i + n_step - 1]), q_t[i + n_step], rescaling, eps)
        td[i] = (q[i] - y).mean()
    out = []
    for i in range(burn_in + learning, E):
        w = td[i - learning + 1:i + 1]
        w = np.abs(w) if metric == "abs" else w ** 2
        out.append(eta * w.max() + (1 - eta) * w.mean())
    return np.asarray(out, np.float64)


def policy_params(O, A, H, seed):
    """{net: state dict} of the four nets in NETS, float32, uniform in +-1 / sqrt(fan-in)."""
    rng = np.random.default_rng(seed)
    out = {}
    for k, name in enumerate(NETS):
        I = O + (A if k >= 2 else 0)
        u = lambda shape, fan: rng.uniform(-1, 1, shape).astype(np.float32) / np.sqrt(fan)  # noqa: E731
        out[name] = {"l1.weight": u((H, I), I), "l1.bias": u(H, I), "l2.weight_ih": u((4 * H, H), H),
                     "l2.weight_hh": u((4 * H, H), H), "l2.bias_ih": u(4 * H, H), "l2.bias_hh": u(4 * H, H),
                     "l3.weight": u((A, H), H), "l3.bias": u(A, H)}
    return out


def policy_step(P, obs, state):
    """Actor.run's step in float64 (P: {net: float64 weights}): obs [N,O], state [4,2,N,H] before -> (mu, state
    after)."""
    new = np.empty_like(state)

    def run(k, x, critic):
        sv = lo.net_forward(P[NETS[k]], x[None], state[k, 0], state[k, 1], critic=critic)
        new[k, 0], new[k, 1] = sv["hs"][1], sv["cs"][1]
        return sv["out"][0]
    mu = run(0, obs, False)
    mu_t = run(1, obs, False)
    run(2, np.concatenate((obs, mu), 1), True)
    run(3, np.concatenate((obs, mu_t), 1), True)
    return mu, new

"""Float64 restatement of the actors' exploration noise (include/r2d2_b200.h r2d2_exploration) on top of
oracle/target_noise's Philox: key = (seed, actor id), counter = (a >> 2, t_lo, t_hi, 1); words (x0, x1) serve a % 4 in
{0, 1} and (x2, x3) serve {2, 3}; z = sqrt(-2 ln u_a) {cos, sin}(2 pi u_b).  Test infrastructure only."""
import numpy as np

from oracle import target_noise as tn


def words(actor_ids, step, n_actions, seed):
    """(x_a, x_b) uint32 [N, A]: the two Philox words each element's Box-Muller pair reads."""
    ids = np.asarray(list(actor_ids), np.uint64)[:, None]
    a = np.arange(n_actions, dtype=np.uint64)[None, :]
    z = np.zeros((len(ids), n_actions), np.uint64)
    x = tn.philox4x32_10((z + (a >> np.uint64(2)), z + np.uint64(step & 0xFFFFFFFF), z + np.uint64(step >> 32),
                          z + np.uint64(1)), (z + np.uint64(seed), z + ids))
    upper = (a & np.uint64(2)) != 0
    return np.where(upper, x[2], x[0]), np.where(upper, x[3], x[1])


def normal(actor_ids, step, n_actions, seed):
    """float64 z [N, A]."""
    wa, wb = words(actor_ids, step, n_actions, seed)
    rad = np.sqrt(-2.0 * np.log(tn.unit_open(wa)))
    odd = (np.arange(n_actions) & 1).astype(bool)[None, :]
    ub = tn.unit_open(wb)
    return rad * np.where(odd, np.sin(2.0 * np.pi * ub), np.cos(2.0 * np.pi * ub))


def run(mu, sigma, actor_ids, seed, mode, theta=0.15, resets=()):
    """float64 actions of T steps: mu [T, N, A], sigma [N]; resets: {step: lanes whose episode begins at that step}
    (OU's x is zero before that step's update).  Step t draws at counter t."""
    mu = np.asarray(mu, np.float64)
    T, N, A = mu.shape
    sig = np.asarray(sigma, np.float64)[:, None]
    x = np.zeros((N, A))
    out = np.empty_like(mu)
    resets = dict(resets)
    for t in range(T):
        x[list(resets.get(t, ()))] = 0.0
        noise = sig * normal(actor_ids, t, A, seed)
        if mode == "ou":
            x = (1.0 - theta) * x + noise
            noise = x
        out[t] = np.clip(mu[t] + noise, -1.0, 1.0)
    return out

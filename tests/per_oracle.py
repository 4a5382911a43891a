"""Float64 restatement of the importance-weighted critic loss (prioritized replay), on top of oracle/learner_oracle.py.

The weighted loss is sum_b w_b sum_{i,a} (q - y)^2 / (L*B*A); its gradient dq = 2 w_b (q - y) / (L*B*A).  td_sq and the
priorities stay unweighted.  `weighted_iteration` runs OracleLearner.iteration with that loss in place of the
unweighted one.
"""
import numpy as np

from oracle import learner_oracle as lo

_UNWEIGHTED_TD = lo.td_targets_and_priorities


def weighted_td(is_weight):
    def td(q, q_next, rew, term, *, burn_in, learning, n_step, gamma, eta=0.9):
        y, _, _, td_sq, prio = _UNWEIGHTED_TD(q, q_next, rew, term, burn_in=burn_in, learning=learning,
                                              n_step=n_step, gamma=gamma, eta=eta)
        w = np.asarray(is_weight, q.dtype).reshape(1, -1, 1)
        diff = q - y
        loss = float(np.sum(w * diff * diff) / diff.size)
        dq = 2.0 * w * diff / diff.size
        return y, loss, dq, td_sq, prio
    return td


def weighted_iteration(learner, batch, is_weight, **kw):
    lo.td_targets_and_priorities = weighted_td(is_weight)
    try:
        return learner.iteration(batch, **kw)
    finally:
        lo.td_targets_and_priorities = _UNWEIGHTED_TD

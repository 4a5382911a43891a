"""Float64 restatement of the learner's optional optimiser extras, on top of oracle/learner_oracle.py (unchanged).

- Gradient-norm clipping goes through OracleLearner.iteration's grad_hook: g <- g * min(1, M / (N + 1e-6)) with N the
  L2 norm over the net's whole gradient block, as torch.nn.utils.clip_grad_norm_(net.parameters(), M) does.
- The Polyak target update is a subclass: on the iterations of the hard copy the targets become
  target (1 - tau) + tau * param', param' the post-Adam weights (utils.soft_update).
"""
import numpy as np

from oracle import learner_oracle as lo


def grad_norm(grads):
    return float(np.sqrt(sum(float(np.sum(np.square(grads[k], dtype=np.float64))) for k in lo.PARAM_KEYS)))


class ClipHook:
    """grad_hook that clips each net's gradient to `max_norm` (0 = off) and records the pre-clip norms."""

    def __init__(self, max_norm):
        self.max_norm = max_norm
        self.norms = {}

    def __call__(self, net, grads):
        n = grad_norm(grads)
        self.norms[net] = n
        if self.max_norm > 0:
            c = min(1.0, self.max_norm / (n + 1e-6))
            for k in lo.PARAM_KEYS:
                grads[k] *= c


class PolyakOracle(lo.OracleLearner):
    """OracleLearner with target_tau: the base class copies the nets into the targets on update iterations, and the
    copy is replaced here by the blend of the previous targets with it."""

    def __init__(self, *args, target_tau=1.0, **kw):
        super().__init__(*args, **kw)
        self.target_tau = target_tau

    def iteration(self, batch, keep=True, grad_hook=None):
        old = (self.target_actor, self.target_critic)
        out = super().iteration(batch, keep=keep, grad_hook=grad_hook)
        if self.step_count % self.target_interval == 0:
            t = self.target_tau
            self.target_actor = {k: old[0][k] * (1.0 - t) + self.actor[k] * t for k in lo.PARAM_KEYS}
            self.target_critic = {k: old[1][k] * (1.0 - t) + self.critic[k] * t for k in lo.PARAM_KEYS}
        return out

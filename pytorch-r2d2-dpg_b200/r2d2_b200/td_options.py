"""The n-step target and priority options (published R2D2's, absent from the reference), in one place.

    value_rescaling  "reference" (default): y = h0(R + gamma^n (1-d) Q'), h0(x) = sign(x)(sqrt(|x|+1) - 1), the reference's
                     utils.py:20-21 - no eps x term, no inverse on the bootstrap;
                     "invertible": y = h_eps(R + gamma^n (1-d) h_eps^-1(Q')), h_eps(x) = h0(x) + eps x.
    rescaling_eps    eps in [0, 1], default 1e-3 (R2D2's); the reference rescaling ignores it.
    priority_metric  "squared" (default): eta max + (1-eta) mean of the squared TD errors (utils.py:17-18);
                     "abs": of the absolute ones (R2D2's; per time step the RMS over the actions, |delta| at one action).

The drop-in learner, the drop-in Actor and ActorPool all read them from the environment through `from_environ`, so every
process of one r2d2.py launch uses the same settings: a replay filled with squared-error priorities and drained by an
abs-priority learner would mix units.  A value that is not one of the allowed ones raises instead of falling back to the
default.
"""
from __future__ import annotations

import math
import os
from dataclasses import dataclass

RESCALINGS = ("reference", "invertible")      # index = R2D2_RESCALE_* of include/r2d2_b200.h
METRICS = ("squared", "abs")                  # index = R2D2_PRIORITY_*
DEFAULT_EPS = 1e-3

ENV_RESCALING = "R2D2_VALUE_RESCALING"
ENV_EPS = "R2D2_RESCALING_EPS"
ENV_METRIC = "R2D2_PRIORITY_METRIC"


def validate(value_rescaling, rescaling_eps, priority_metric):
    """Raise ValueError unless the three settings are allowed values."""
    if value_rescaling not in RESCALINGS:
        raise ValueError("value_rescaling=%r: allowed values are %s" % (value_rescaling, ", ".join(RESCALINGS)))
    if priority_metric not in METRICS:
        raise ValueError("priority_metric=%r: allowed values are %s" % (priority_metric, ", ".join(METRICS)))
    if isinstance(rescaling_eps, bool) or not isinstance(rescaling_eps, (int, float)) or \
            not (math.isfinite(rescaling_eps) and 0.0 <= rescaling_eps <= 1.0):
        raise ValueError("rescaling_eps=%r: allowed values are finite numbers in [0, 1]" % (rescaling_eps,))


@dataclass(frozen=True)
class TdOptions:
    value_rescaling: str = "reference"
    rescaling_eps: float = DEFAULT_EPS
    priority_metric: str = "squared"

    def __post_init__(self):
        validate(self.value_rescaling, self.rescaling_eps, self.priority_metric)

    @property
    def is_default(self) -> bool:
        """The reference's target and priorities (eps does not matter to the reference rescaling)."""
        return self.value_rescaling == "reference" and self.priority_metric == "squared"

    def native(self):
        """(rescaling, eps, priority_metric) as the library's r2d2_td_options fields."""
        return RESCALINGS.index(self.value_rescaling), float(self.rescaling_eps), METRICS.index(self.priority_metric)


def from_environ(environ=None) -> TdOptions:
    """R2D2_VALUE_RESCALING=reference|invertible, R2D2_RESCALING_EPS (default 1e-3), R2D2_PRIORITY_METRIC=squared|abs."""
    env = os.environ if environ is None else environ
    rescaling = env.get(ENV_RESCALING, "reference")
    metric = env.get(ENV_METRIC, "squared")
    if rescaling not in RESCALINGS:
        raise ValueError("%s=%r: allowed values are %s" % (ENV_RESCALING, rescaling, ", ".join(RESCALINGS)))
    if metric not in METRICS:
        raise ValueError("%s=%r: allowed values are %s" % (ENV_METRIC, metric, ", ".join(METRICS)))
    raw = env.get(ENV_EPS)
    eps = DEFAULT_EPS
    if raw is not None:
        try:
            eps = float(raw)
        except ValueError:
            eps = None
        if eps is None or not (math.isfinite(eps) and 0.0 <= eps <= 1.0):
            raise ValueError("%s=%r: allowed values are finite numbers in [0, 1]" % (ENV_EPS, raw))
    return TdOptions(rescaling, eps, metric)

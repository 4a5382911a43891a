"""Actor exploration options (absent from the reference, which adds N(0, 0.3) on the host), read from the environment in
one place, and the host restatement of the noise the policy-step kernel draws (include/r2d2_b200.h r2d2_exploration).

    R2D2_EXPLORATION             reference (default): the reference's host noise, unchanged;
                                 gaussian: a = clip(mu + sigma_i z, -1, 1);
                                 ou: x <- (1 - theta) x + sigma_i z, a = clip(mu + x, -1, 1), x per actor and action,
                                 zero at every episode start
    R2D2_EXPLORATION_SIGMA       sigma_max, finite >= 0 (default 0.3)
    R2D2_EXPLORATION_SIGMA_MIN   sigma_min (default sigma_max); when it differs, 0 < sigma_min <= sigma_max
    R2D2_EXPLORATION_ACTORS      N >= 1, required when sigma_min != sigma_max: actor i gets
                                 sigma_i = sigma_max (sigma_min / sigma_max)^(i / (N - 1)) (Ape-X's log-spaced schedule),
                                 in float64 rounded to float32 once; an actor id >= N raises
    R2D2_EXPLORATION_OU_THETA    theta in (0, 1] (default 0.15), ou only
    R2D2_EXPLORATION_SEED        integer in [0, 2**32) (default 0)

z for actor i, action a at the actor's env step t (its 0-based count since the process started, across episodes) comes
from Philox4x32-10 with key (seed, i) and counter (a >> 2, t mod 2**32, t >> 32, 1), so actor i draws the same noise
in a drop-in Actor, in any ActorPool lane and on the GPU or the host.  A malformed value raises and names the allowed
ones; under `reference` any other R2D2_EXPLORATION_* variable raises, so no setting is silently ignored.

`HostNoise` is the numpy restatement the CPU steppers and the drop-in Actor use.  Its Philox words are the kernel's bit
for bit and its fp32 operation order is the kernel's; z differs from the kernel's by at most the error of CUDA's logf
and sincospif (1 ulp each, documented), which bounds |z_host - z_device| by 4 ulp of z.
"""
from __future__ import annotations

import math
import os
from dataclasses import dataclass

import numpy as np

MODES = ("reference", "gaussian", "ou")      # gaussian, ou: index - 1 = R2D2_EXPLORATION_* of include/r2d2_b200.h

ENV_MODE = "R2D2_EXPLORATION"
ENV_SIGMA = "R2D2_EXPLORATION_SIGMA"
ENV_SIGMA_MIN = "R2D2_EXPLORATION_SIGMA_MIN"
ENV_ACTORS = "R2D2_EXPLORATION_ACTORS"
ENV_THETA = "R2D2_EXPLORATION_OU_THETA"
ENV_SEED = "R2D2_EXPLORATION_SEED"
ENV_OPTIONS = (ENV_SIGMA, ENV_SIGMA_MIN, ENV_ACTORS, ENV_THETA, ENV_SEED)

DEFAULT_SIGMA = 0.3
DEFAULT_THETA = 0.15


@dataclass(frozen=True)
class Exploration:
    mode: str = "reference"
    sigma: float = DEFAULT_SIGMA          # sigma_max
    sigma_min: float | None = None        # None: sigma_max
    actors: int | None = None             # N of the schedule
    theta: float = DEFAULT_THETA
    seed: int = 0

    def __post_init__(self):
        if self.mode not in MODES:
            raise ValueError("mode=%r: allowed values are %s" % (self.mode, ", ".join(MODES)))
        if not (_real(self.sigma) and self.sigma >= 0.0):
            raise ValueError("sigma=%r: allowed values are finite numbers >= 0" % (self.sigma,))
        if self.sigma_min is not None and self.sigma_min != self.sigma and \
                not (_real(self.sigma_min) and 0.0 < self.sigma_min <= self.sigma):
            raise ValueError("sigma_min=%r: allowed values are finite numbers in (0, sigma=%r]"
                             % (self.sigma_min, self.sigma))
        if self.actors is not None and (isinstance(self.actors, bool) or not isinstance(self.actors, int)
                                        or self.actors < 1):
            raise ValueError("actors=%r: allowed values are integers >= 1" % (self.actors,))
        if self.actors is None and self.sigma_min is not None and self.sigma_min != self.sigma:
            raise ValueError("sigma_min=%r differs from sigma=%r: the schedule needs the number of actors (%s)"
                             % (self.sigma_min, self.sigma, ENV_ACTORS))
        if not (_real(self.theta) and 0.0 < self.theta <= 1.0):
            raise ValueError("theta=%r: allowed values are numbers in (0, 1]" % (self.theta,))
        if isinstance(self.seed, bool) or not isinstance(self.seed, int) or not 0 <= self.seed < 2 ** 32:
            raise ValueError("seed=%r: allowed values are integers in [0, 2**32)" % (self.seed,))

    @property
    def kind(self) -> int:
        """R2D2_EXPLORATION_GAUSSIAN (0) or R2D2_EXPLORATION_OU (1); only for gaussian and ou."""
        return MODES.index(self.mode) - 1

    @property
    def one_minus_theta(self) -> np.float32:
        """fl32(1 - theta), the OU decay the kernel and the host both read."""
        return np.float32(1.0 - self.theta)

    def sigmas(self, actor_ids) -> np.ndarray:
        """float32 sigma_i of these actor ids (the log-spaced schedule, or sigma_max for every id)."""
        ids = np.asarray(list(actor_ids), np.int64)
        if np.any(ids < 0) or np.any(ids >= 2 ** 32):
            raise ValueError("actor ids must be in [0, 2**32): %s" % ids[(ids < 0) | (ids >= 2 ** 32)])
        if self.actors is not None and np.any(ids >= self.actors):
            raise ValueError("actor id %d >= %s=%d: the schedule covers ids 0 .. %d"
                             % (int(ids[ids >= self.actors][0]), ENV_ACTORS, self.actors, self.actors - 1))
        lo = self.sigma if self.sigma_min is None else self.sigma_min
        if lo == self.sigma or self.actors == 1:
            return np.full(len(ids), self.sigma, np.float32)
        f = ids.astype(np.float64) / (self.actors - 1)
        s = float(self.sigma) * (float(lo) / float(self.sigma)) ** f
        s = np.where(ids == self.actors - 1, float(lo), s)        # the far end is sigma_min exactly
        return s.astype(np.float32)


def _real(v) -> bool:
    return not isinstance(v, bool) and isinstance(v, (int, float, np.floating)) and math.isfinite(v)


def from_environ(environ=None) -> Exploration:
    """The options of the R2D2_EXPLORATION* variables (module docstring)."""
    env = os.environ if environ is None else environ
    mode = env.get(ENV_MODE, "reference")
    if mode not in MODES:
        raise ValueError("%s=%r: allowed values are %s" % (ENV_MODE, mode, ", ".join(MODES)))
    if mode == "reference":
        given = [k for k in ENV_OPTIONS if k in env]
        if given:
            raise ValueError("%s is set but %s=reference applies no such setting: allowed values of %s with it are "
                             "gaussian, ou" % (", ".join(given), ENV_MODE, ENV_MODE))
        return Exploration()
    if mode != "ou" and ENV_THETA in env:
        raise ValueError("%s=%r is set but %s=%s: it is allowed with %s=ou only"
                         % (ENV_THETA, env[ENV_THETA], ENV_MODE, mode, ENV_MODE))

    def real(name, default, ok, allowed):
        raw = env.get(name)
        if raw is None:
            return default
        try:
            v = float(raw)
        except ValueError:
            v = None
        if v is None or not (math.isfinite(v) and ok(v)):
            raise ValueError("%s=%r: allowed values are %s" % (name, raw, allowed))
        return v

    def integer(name, default, lo, hi, allowed):
        raw = env.get(name)
        if raw is None:
            return default
        try:
            v = int(raw)
        except ValueError:
            v = None
        if v is None or not lo <= v < hi:
            raise ValueError("%s=%r: allowed values are %s" % (name, raw, allowed))
        return v

    sigma = real(ENV_SIGMA, DEFAULT_SIGMA, lambda v: v >= 0.0, "finite numbers >= 0")
    sigma_min = real(ENV_SIGMA_MIN, None, lambda v: v == sigma or 0.0 < v <= sigma,
                     "finite numbers in (0, %s=%r]" % (ENV_SIGMA, sigma))
    actors = integer(ENV_ACTORS, None, 1, 2 ** 32, "integers >= 1")
    if actors is None and sigma_min is not None and sigma_min != sigma:
        raise ValueError("%s=%r differs from %s=%r: %s (allowed values: integers >= 1) is required"
                         % (ENV_SIGMA_MIN, env[ENV_SIGMA_MIN], ENV_SIGMA, sigma, ENV_ACTORS))
    theta = real(ENV_THETA, DEFAULT_THETA, lambda v: 0.0 < v <= 1.0, "numbers in (0, 1]")
    seed = integer(ENV_SEED, 0, 0, 2 ** 32, "integers in [0, 2**32)")
    return Exploration(mode, sigma, sigma_min, actors, theta, seed)


# ------------------------------------------------------------------------------------------------ the generator
_M0, _M1, _W0, _W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
_MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """Philox4x32-10 in numpy uint64 arithmetic.  ctr: four uint32 arrays (or scalars), key: two; broadcast together.
    Returns the four output words as uint32 arrays."""
    c = [np.asarray(x, np.uint64) & _MASK for x in ctr]
    k0, k1 = (np.asarray(x, np.uint64) & _MASK for x in key)
    for r in range(10):
        if r:
            k0, k1 = (k0 + np.uint64(_W0)) & _MASK, (k1 + np.uint64(_W1)) & _MASK
        p0 = np.uint64(_M0) * c[0]
        p1 = np.uint64(_M1) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _MASK, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _MASK]
    return [x.astype(np.uint32) for x in c]


def _sincospi(y):
    """(sin(pi y), cos(pi y)) in float64 for float64 y, exact at multiples of 1/2 (as sincospif is)."""
    q = np.rint(2.0 * y)
    r = np.pi * (y - 0.5 * q)                            # y - q/2 is exact: |.| <= 1/4
    s, c = np.sin(r), np.cos(r)
    k = q.astype(np.int64) & 3
    sin = np.choose(k, [s, c, -s, -c])
    cos = np.choose(k, [c, -s, -c, s])
    return sin, cos


def normal(actor_ids, step, n_actions, seed):
    """float32 z [len(actor_ids), n_actions] of the kernel's stream (key (seed, id), counter (a >> 2, t_lo, t_hi, 1))
    at env step `step`: u = (2 (x >> 9) + 1) 2^-24 (exact in fp32); rad = sqrtf(-2 logf(u_a)); z = fl(rad cospi(2 u_b))
    for even a % 4 and fl(rad sinpi(2 u_b)) for odd, with logf and sincospif taken correctly rounded."""
    ids = np.asarray(list(actor_ids), np.uint64)[:, None]
    a = np.arange(n_actions, dtype=np.uint64)[None, :]
    step = int(step)
    z0 = np.zeros((len(ids), n_actions), np.uint64)
    x = philox4x32_10((z0 + (a >> np.uint64(2)), z0 + np.uint64(step & 0xFFFFFFFF), z0 + np.uint64(step >> 32),
                       z0 + np.uint64(1)), (z0 + np.uint64(seed), z0 + ids))
    upper = ((a & np.uint64(2)) != 0)
    wa, wb = np.where(upper, x[2], x[0]), np.where(upper, x[3], x[1])
    ua = ((2 * (wa >> np.uint32(9)).astype(np.int64) + 1) * 2.0 ** -24).astype(np.float32)
    ub = ((2 * (wb >> np.uint32(9)).astype(np.int64) + 1) * 2.0 ** -24).astype(np.float32)
    rad = np.sqrt(np.float32(-2.0) * np.log(ua.astype(np.float64)).astype(np.float32))
    s, c = _sincospi(2.0 * ub.astype(np.float64))
    odd = (a & np.uint64(1)) != 0
    return (rad * np.where(odd, s, c).astype(np.float32)).astype(np.float32)


class HostNoise:
    """The kernel's exploration on the host for a fixed list of actor ids (one lane each): `actions(mu, step)` ->
    float32 clip(mu + noise) in the kernel's fp32 operation order; `reset(lanes)` zeroes the lanes' OU state."""

    def __init__(self, options: Exploration, actor_ids, n_actions):
        if options.mode == "reference":
            raise ValueError("HostNoise is for the gaussian and ou modes; reference noise stays with its caller")
        self.options = options
        self.actor_ids = list(actor_ids)
        self.sigma = options.sigmas(self.actor_ids)[:, None]
        self.x = np.zeros((len(self.actor_ids), n_actions), np.float32) if options.mode == "ou" else None
        self.n_actions = n_actions

    def reset(self, lanes):
        if self.x is not None:
            self.x[list(lanes)] = 0.0

    def actions(self, mu, step):
        z = normal(self.actor_ids, step, self.n_actions, self.options.seed)
        noise = self.sigma * z                                           # fp32 products, rounded once each
        if self.x is not None:
            self.x = self.options.one_minus_theta * self.x + noise
            noise = self.x
        return np.clip(np.asarray(mu, np.float32) + noise, np.float32(-1), np.float32(1)).astype(np.float32)

"""TD3's target options of the drop-in learner (absent from the reference), read from the environment in one place.

    R2D2_TWIN_CRITIC         0 (default) or 1: a second critic and target critic, bootstrap from the minimum of the two
    R2D2_TARGET_NOISE        sigma, finite >= 0 (default 0 = off): target policy smoothing clip(sigma z, -c, c)
    R2D2_TARGET_NOISE_CLIP   c, finite > 0 (default 0.5)
    R2D2_TARGET_NOISE_SEED   integer in [0, 2**32) (default 0): the noise key is (seed, rank)

TD3's usual setting: R2D2_TWIN_CRITIC=1 R2D2_TARGET_NOISE=0.2 R2D2_TARGET_NOISE_CLIP=0.5 with R2D2_TARGET_TAU=0.005
R2D2_TARGET_INTERVAL=1.  A value that is not an allowed one raises and names the allowed ones.
"""
from __future__ import annotations

import math
import os

ENV_TWIN = "R2D2_TWIN_CRITIC"
ENV_NOISE = "R2D2_TARGET_NOISE"
ENV_CLIP = "R2D2_TARGET_NOISE_CLIP"
ENV_SEED = "R2D2_TARGET_NOISE_SEED"


def from_environ(environ=None) -> dict:
    """PathConfig keyword arguments twin_critic, target_noise, target_noise_clip, target_noise_seed."""
    env = os.environ if environ is None else environ
    twin = env.get(ENV_TWIN, "0")
    if twin not in ("0", "1"):
        raise ValueError("%s=%r: allowed values are 0, 1" % (ENV_TWIN, twin))

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

    sigma = real(ENV_NOISE, 0.0, lambda v: v >= 0.0, "finite numbers >= 0 (0 = off)")
    clip = real(ENV_CLIP, 0.5, lambda v: v > 0.0, "finite numbers > 0")
    raw = env.get(ENV_SEED, "0")
    try:
        seed = int(raw)
    except ValueError:
        seed = -1
    if not 0 <= seed < 2 ** 32:
        raise ValueError("%s=%r: allowed values are integers in [0, 2**32)" % (ENV_SEED, raw))
    return dict(twin_critic=twin == "1", target_noise=sigma, target_noise_clip=clip, target_noise_seed=seed)

"""Observation normalisation (off by default): running per-feature mean and variance of the ingested observation rows,
applied where the nets read the observation - the replay gather, the actors' step kernel, the actor-priority chains.

One definition everywhere (include/r2d2_b200.h, r2d2_obs_norm_merge): float64 statistics n, mean [O], M2 [O] over every
ingested row that is no pad row and holds only finite values, merged with Chan's parallel formula; the fp32 pair
mean_f = (float) mean, inv_std_f = (float)(1 / sqrt(M2 / n + 1e-8)); x_hat = clamp(fl(fl(x - mean_f) * inv_std_f), -c, c)
with NaN passing through.  Only observations are normalised; the replay, its snapshots and its export stay raw.

`ObsNormStats` holds the learner's device statistics: `running` (what the gathers read, through mean_f / inv_std_f) and
`pending` (this rank's ingests since the last exchange).  The statistics change only at `exchange()`, which the training
loop calls at points every rank reaches equally often (r2d2_b200.run_loop): data-parallel ranks all-gather their pending
blocks there and merge them in rank order, so every rank ends with the same bits.
"""
from __future__ import annotations

import math
import os
from ctypes import c_void_p

import numpy as np
import torch

DEFAULT_CLIP = 5.0


def from_environ(env=None):
    """(enabled, clip) from R2D2_OBS_NORM=0|1 (default 0) and R2D2_OBS_NORM_CLIP (finite and > 0, default 5)."""
    env = os.environ if env is None else env
    v = env.get("R2D2_OBS_NORM", "0")
    if v not in ("0", "1"):
        raise ValueError("R2D2_OBS_NORM must be 0 or 1, got %r" % (v,))
    c = env.get("R2D2_OBS_NORM_CLIP", str(DEFAULT_CLIP))
    try:
        clip = float(c)
    except (TypeError, ValueError):
        clip = float("nan")
    if not (math.isfinite(clip) and clip > 0):
        raise ValueError("R2D2_OBS_NORM_CLIP must be a finite number > 0, got %r" % (c,))
    return v == "1", clip


def validate_clip(clip):
    if isinstance(clip, bool) or not isinstance(clip, (int, float, np.floating, np.integer)) or not (
            math.isfinite(clip) and clip > 0):
        raise ValueError("obs_norm_clip must be finite and > 0, got %r" % (clip,))


def normalize_torch(x: torch.Tensor, mean_f: torch.Tensor, inv_std_f: torch.Tensor, clip: float) -> torch.Tensor:
    """The transform in torch fp32 (sub, mul, clamp: the kernels' bits), for the drop-in Actor."""
    return torch.clamp((x.float() - mean_f.to(x.device)) * inv_std_f.to(x.device), -float(clip), float(clip))


class ObsNormStats:
    """Device statistics of one learner rank: running / pending moment blocks [1 + 2 O] (float64), the fp32 pair the
    kernels read, and the scratch block an ingest call writes its moments into."""

    def __init__(self, obs: int, clip: float, device):
        from . import native as nv
        validate_clip(clip)
        self.lib, self.O, self.clip, self.device = nv.lib(), int(obs), float(clip), torch.device(device)
        z = lambda: torch.zeros(1 + 2 * self.O, dtype=torch.float64, device=self.device)  # noqa: E731
        self.running, self.pending, self.ingest_block = z(), z(), z()
        self.mean_f = torch.zeros(self.O, dtype=torch.float32, device=self.device)
        self.inv_std_f = torch.ones(self.O, dtype=torch.float32, device=self.device)
        self.nonfinite_rows = 0        # ingested non-pad rows left out for a NaN or +-inf value
        self.dist = None               # torch.distributed, set by LearnerEngine.enable_data_parallel

    def _merge(self, into: torch.Tensor, blocks: torch.Tensor, fp32: bool):
        from . import native as nv
        W = blocks.shape[0]
        mf = c_void_p(self.mean_f.data_ptr()) if fp32 else None
        sf = c_void_p(self.inv_std_f.data_ptr()) if fp32 else None
        nv.check(self.lib.r2d2_obs_norm_merge(c_void_p(into.data_ptr()), c_void_p(blocks.data_ptr()), W, self.O, mf, sf,
                                              nv.current_stream()))

    def add_ingest(self, nonfinite: int = 0):
        """Fold the moments the last ingest call wrote into `ingest_block` into `pending` (local, no collective)."""
        self._merge(self.pending, self.ingest_block.view(1, -1), fp32=False)
        self.nonfinite_rows += int(nonfinite)

    def exchange(self, blocks: torch.Tensor | None = None):
        """Merge every rank's pending block into `running` in rank order, rewrite mean_f / inv_std_f and clear `pending`.
        With a process group this all-gathers the pending blocks (a collective); `blocks` [W, 1 + 2 O] gives them
        directly instead (in-process ranks)."""
        if blocks is None:
            if self.dist is not None:
                blocks = torch.empty((self.dist.get_world_size(), 1 + 2 * self.O), dtype=torch.float64,
                                     device=self.device)
                self.dist.all_gather_into_tensor(blocks, self.pending)
            else:
                blocks = self.pending.view(1, -1).clone()
        self._merge(self.running, blocks.contiguous(), fp32=True)
        self.pending.zero_()

    @property
    def count(self) -> float:
        return float(self.running[0].item())

    def state(self) -> dict:
        """The training state's record: on, clip, n, mean, M2 (float64 arrays)."""
        r = self.running.cpu().numpy()
        return {"enabled": True, "clip": self.clip, "n": float(r[0]), "mean": r[1:1 + self.O].copy(),
                "M2": r[1 + self.O:].copy()}

    def load_state(self, st: dict):
        mean, m2 = np.asarray(st["mean"], np.float64), np.asarray(st["M2"], np.float64)
        if mean.shape != (self.O,) or m2.shape != (self.O,):
            raise ValueError("obs_norm statistics of width %r / %r, this engine has obs %d" % (mean.shape, m2.shape, self.O))
        self.running.copy_(torch.as_tensor(np.concatenate([[float(st["n"])], mean, m2])))
        self.pending.zero_()
        # the fp32 pair from the restored statistics: a merge of nothing
        self._merge(self.running, torch.zeros((1, 1 + 2 * self.O), dtype=torch.float64, device=self.device), fp32=True)

    def actor_key(self):
        """model.pt's `obs_norm` entry {mean_f, inv_std_f, clip} (CPU tensors), or None before the first row."""
        if self.count <= 0:
            return None
        return {"mean_f": self.mean_f.detach().cpu().clone(), "inv_std_f": self.inv_std_f.detach().cpu().clone(),
                "clip": self.clip}

"""Host-side orchestration of the native learner path (torch = device memory, streams, NCCL).

`LearnerEngine` owns the flat parameter / gradient / Adam buffers (torch CUDA tensors), exposes them
as `state_dict()`-compatible views with the reference's keys (models.py:17-19), and drives the three
native phases of one learner iteration (learner.py:84-139).  With torch.distributed initialised it
all-reduces the two flat gradient buffers between the phases (SURVEY 8e): nothing else crosses GPUs.

`DeviceReplay` is the per-GPU replay shard (replaces LearnerReplayMemory storage + sampling,
replay_memory.py:67-136) with the sum tree in HBM.
"""
from __future__ import annotations

import math
import numbers
from collections import OrderedDict
from ctypes import byref, c_int, c_longlong, c_size_t, c_void_p
from dataclasses import dataclass

import numpy as np
import torch

from . import metrics as metrics_mod
from . import native as nv
from . import obs_norm as obs_norm_mod
from . import td_options

# PathConfig.replay_state_dtype -> r2d2_replay_options.state_storage
REPLAY_STATE_DTYPES = {"float32": nv.STATE_F32, "float16": nv.STATE_F16}
# PathConfig.replay_state_memory -> r2d2_replay_options.state_memory
REPLAY_STATE_MEMORY = {"device": nv.STATE_MEMORY_DEVICE, "host": nv.STATE_MEMORY_HOST}

PARAM_KEYS = ("l1.weight", "l1.bias", "l2.weight_ih", "l2.weight_hh", "l2.bias_ih", "l2.bias_hh",
              "l3.weight", "l3.bias")


@dataclass
class PathConfig:
    """Hyper-parameters of the path; defaults are the reference's literals (learner.py:29-34,43-49).

    Prioritized replay (not in the reference, whose defaults these are): `priority_exponent` alpha - the replay shard
    samples a start with probability p^alpha / sum p^alpha (published R2D2: 0.9) - and `is_exponent` beta - the critic
    loss weights sequence b by (min_b' P_b' / P_b)^beta, normalised over the batch (R2D2: 0.6).  Both lie in [0, 1].

    Optimiser step (not in the reference either): `target_tau` tau in (0, 1] - on the iterations of the target update
    (every `target_interval` steps) each target net becomes target (1 - tau) + tau * the net's post-Adam weights, like
    the reference's unused utils.soft_update; 1 is the hard copy (DDPG: 0.005 at interval 1).  The library holds tau in
    float32.  `grad_clip_norm` M >= 0 - each net's gradient is scaled by min(1, M / (N + 1e-6)), N its global L2 norm,
    like torch.nn.utils.clip_grad_norm_; 0 is off.

    n-step target and priorities (r2d2_b200.td_options): `value_rescaling` "reference" (the reference's h0 without an
    inverse on the bootstrap) or "invertible" (R2D2's h_eps(R + gamma^n (1-d) h_eps^-1(Q')) with eps = `rescaling_eps`,
    in [0, 1]); `priority_metric` "squared" (the reference's) or "abs" (R2D2's absolute TD errors).

    TD3's target (include/r2d2_b200.h, r2d2_learner_options): `twin_critic` adds a second critic and target critic and
    bootstraps from the minimum of the two target critics; `target_noise` sigma >= 0 (0 = off) smooths the target actor's
    actions with clip(sigma z, -c, c), c = `target_noise_clip` > 0, z keyed on (`target_noise_seed`, rank) and the
    iteration index.  TD3's usual setting: twin, sigma 0.2, c 0.5, target_tau 0.005 at target_interval 1.

    `global_sampling` (data parallel, off by default): the W ranks draw one global batch of W * B sequences from the
    union of their replay shards in proportion to the stored leaves p^alpha, and rank c trains on global draws
    c*B .. c*B+B-1 (DeviceReplay.attach_group).  The engine's batch slots then live in memory every rank maps; at W = 1
    the draws, batches and weights are the local mode's bit for bit.

    `replay_state_dtype` (replay shard, include/r2d2_b200.h r2d2_replay_options): "float32" (default) stores the four
    nets' recurrent states of every row in fp32; "float16" stores them in fp16 - nearly twice the rows in the same HBM -
    rounded once at ingest and widened exactly by the gather, so training sees the fp16-rounded states.  An actor file
    with a finite state of magnitude >= 65520 is refused whole in that mode.

    `replay_state_memory` (replay shard): "device" (default) keeps those states in HBM; "host" keeps them in mapped,
    page-locked host memory while the rest of every row and the sum tree stay in HBM.  The gather then reads each drawn
    sequence's start states over the host link; the batch is bit-identical to the device tier's.

    `obs_norm` (off by default, r2d2_b200.obs_norm): the engine keeps running float64 mean / variance statistics of the
    ingested observation rows (DeviceReplay.add_episodes(obs_norm=...)), and every gather of an attached shard writes
    x_hat = clamp((x - mean) / std, -c, c) into the batch, c = `obs_norm_clip` (> 0, default 5).  Actions, rewards,
    terminals and stored states are not normalised; the replay keeps raw rows.  The statistics change only at
    LearnerEngine.obs_norm.exchange(), which the training loop calls after its ingests (run_loop).

    `metrics` (off by default, r2d2_b200.metrics): the library reduces one record of training statistics per iteration
    on the device into a ring that LearnerEngine.metrics.read() returns; training itself is bit-identical either way."""
    obs: int
    act: int
    hidden: int = 128
    batch: int = 32
    burn_in: int = 20
    learning: int = 40
    n_step: int = 5
    gamma: float = 0.997
    actor_lr: float = 1e-4
    critic_lr: float = 1e-3
    eta: float = 0.9
    target_interval: int = 500
    priority_exponent: float = 1.0
    is_exponent: float = 0.0
    target_tau: float = 1.0
    grad_clip_norm: float = 0.0
    value_rescaling: str = "reference"
    rescaling_eps: float = td_options.DEFAULT_EPS
    priority_metric: str = "squared"
    twin_critic: bool = False
    target_noise: float = 0.0
    target_noise_clip: float = 0.5
    target_noise_seed: int = 0
    global_sampling: bool = False
    replay_state_dtype: str = "float32"
    replay_state_memory: str = "device"
    obs_norm: bool = False
    obs_norm_clip: float = obs_norm_mod.DEFAULT_CLIP
    metrics: bool = False

    def __post_init__(self):
        for name, least in (("burn_in", 0), ("learning", 2), ("n_step", 1)):
            v = getattr(self, name)
            if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or v < least:
                raise ValueError("%s must be an integer >= %d, got %r%s" % (
                    name, least, v, " (the priority series [b:-1:B] of the last batch element drops its last TD step, "
                                    "so a one-step window leaves it empty)" if name == "learning" else ""))
        td_options.validate(self.value_rescaling, self.rescaling_eps, self.priority_metric)
        if not isinstance(self.replay_state_dtype, str) or self.replay_state_dtype not in REPLAY_STATE_DTYPES:
            raise ValueError("replay_state_dtype must be one of %s, got %r" % (", ".join(REPLAY_STATE_DTYPES),
                                                                              self.replay_state_dtype))
        if not isinstance(self.replay_state_memory, str) or self.replay_state_memory not in REPLAY_STATE_MEMORY:
            raise ValueError("replay_state_memory must be one of %s, got %r" % (", ".join(REPLAY_STATE_MEMORY),
                                                                               self.replay_state_memory))
        obs_norm_mod.validate_clip(self.obs_norm_clip)
        for name in ("twin_critic", "global_sampling", "obs_norm", "metrics"):
            if not isinstance(getattr(self, name), bool):
                raise ValueError("%s must be True or False, got %r" % (name, getattr(self, name)))
        for name, lo_ok in (("target_noise", lambda v: v >= 0.0), ("target_noise_clip", lambda v: v > 0.0)):
            v = getattr(self, name)
            if isinstance(v, bool) or not isinstance(v, numbers.Real) or not (math.isfinite(v) and lo_ok(v)):
                raise ValueError("%s must be finite and %s, got %r" % (name, ">= 0 (0 = off)" if name == "target_noise"
                                                                        else "> 0", v))
        s = self.target_noise_seed
        if isinstance(s, bool) or not isinstance(s, (int, np.integer)) or not 0 <= s < 2 ** 32:
            raise ValueError("target_noise_seed must be an integer in [0, 2**32), got %r" % (s,))
        for name in ("priority_exponent", "is_exponent"):
            v = getattr(self, name)
            if not 0.0 <= v <= 1.0:
                raise ValueError("%s must lie in [0, 1], got %r" % (name, v))
        if not 0.0 < self.target_tau <= 1.0:
            raise ValueError("target_tau must lie in (0, 1], got %r" % (self.target_tau,))
        if not (0.0 <= self.grad_clip_norm and math.isfinite(self.grad_clip_norm)):
            raise ValueError("grad_clip_norm must be finite and >= 0 (0 = off), got %r" % (self.grad_clip_norm,))

    @property
    def rows(self) -> int:
        return self.burn_in + self.learning + self.n_step


def param_shapes(cfg: PathConfig, critic: bool):
    H, A = cfg.hidden, cfg.act
    I = cfg.obs + (cfg.act if critic else 0)
    return OrderedDict([("l1.weight", (H, I)), ("l1.bias", (H,)), ("l2.weight_ih", (4 * H, H)),
                        ("l2.weight_hh", (4 * H, H)), ("l2.bias_ih", (4 * H,)), ("l2.bias_hh", (4 * H,)),
                        ("l3.weight", (A, H)), ("l3.bias", (A,))])


def flat_views(flat: torch.Tensor, cfg: PathConfig, critic: bool):
    """state_dict-ordered views into a flat parameter block (no copies)."""
    out, off = OrderedDict(), 0
    for k, shp in param_shapes(cfg, critic).items():
        n = int(np.prod(shp))
        out[k] = flat[off:off + n].view(shp)
        off += n
    assert off == flat.numel()
    return out


def init_reference_params(cfg: PathConfig, critic: bool, generator: torch.Generator | None = None):
    """Fresh parameters with the reference's distributions (models.py:8-11,21-25): fan-in uniform keyed
    on out_features for l1 / LSTM weights, LSTMCell-default U(+-1/sqrt(H)) biases, Linear-default l1 bias,
    l3 U(+-3e-3) / 3e-4.  (Seed-for-seed identity with torch's module constructors is not needed here;
    parity tests load the reference's own tensors.)"""
    H = cfg.hidden
    shapes = param_shapes(cfg, critic)
    u = lambda shp, b: (torch.rand(shp, generator=generator) * 2 - 1) * b  # noqa: E731
    I = shapes["l1.weight"][1]
    p = OrderedDict()
    p["l1.weight"] = u(shapes["l1.weight"], 1.0 / np.sqrt(H))
    p["l1.bias"] = u(shapes["l1.bias"], 1.0 / np.sqrt(I))
    p["l2.weight_ih"] = u(shapes["l2.weight_ih"], 1.0 / np.sqrt(4 * H))
    p["l2.weight_hh"] = u(shapes["l2.weight_hh"], 1.0 / np.sqrt(4 * H))
    p["l2.bias_ih"] = u(shapes["l2.bias_ih"], 1.0 / np.sqrt(H))
    p["l2.bias_hh"] = u(shapes["l2.bias_hh"], 1.0 / np.sqrt(H))
    p["l3.weight"] = u(shapes["l3.weight"], 3e-3)
    p["l3.bias"] = torch.full(shapes["l3.bias"], 3e-4)
    return p


class LearnerEngine:
    def __init__(self, cfg: PathConfig, device=None, seed: int = 1):
        if not torch.cuda.is_available():
            raise nv.NativeError("LearnerEngine needs a CUDA device (H100); there is no CPU fallback")
        import os
        # data-parallel gradient exchange: "peer" (default: the library's own kernels over NVLink peer memory, in the
        # learner's stream) or "defer" (NCCL all-reduces on a side stream, the actor's waited for one critic phase later;
        # also the fallback when no peer-mapped buffer can be set up)
        self._dp_mode = os.environ.get("R2D2_DP_MODE", "peer")
        if self._dp_mode not in ("peer", "defer"):
            raise nv.NativeError("R2D2_DP_MODE=%r: the gradient exchange mode is 'peer' (default) or 'defer'"
                                 % self._dp_mode)
        self.lib = nv.lib()
        self.cfg = cfg
        self._pending_finish = False          # a deferred phase 3 (data parallel), see step() / flush()
        self._h = None
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        torch.cuda.set_device(self.device)
        na = sum(int(np.prod(s)) for s in param_shapes(cfg, False).values())
        nc = sum(int(np.prod(s)) for s in param_shapes(cfg, True).values())
        z = lambda n: torch.zeros(n, dtype=torch.float32, device=self.device)  # noqa: E731
        # twin critic: every critic block is [critic 1 | pad | critic 2 | pad], critic 2 at P' = P rounded up to 64 floats
        # (include/r2d2_b200.h); views("critic") stays critic 1
        self._n_critic = nc
        self._critic2_off = -(-nc // 64) * 64 if cfg.twin_critic else 0
        ncb = 2 * self._critic2_off if cfg.twin_critic else nc
        self.flat = {"actor": z(na), "critic": z(ncb), "target_actor": z(na), "target_critic": z(ncb)}
        self.grads = {"actor": z(na), "critic": z(ncb)}
        self.exp_avg = {"actor": z(na), "critic": z(ncb)}
        self.exp_avg_sq = {"actor": z(na), "critic": z(ncb)}
        g = torch.Generator().manual_seed(seed)
        self.load_state_dicts(init_reference_params(cfg, False, g), init_reference_params(cfg, True, g))
        if cfg.twin_critic:                      # drawn after the four reference nets: their values do not move
            c2 = init_reference_params(cfg, True, g)
            self.load_state_dicts(None, None, critic2=c2, target_critic2=c2)
        c = nv.LearnerConfig(cfg.obs, cfg.act, cfg.hidden, cfg.batch, cfg.burn_in, cfg.learning, cfg.n_step,
                             cfg.gamma, cfg.actor_lr, cfg.critic_lr, cfg.eta, cfg.target_interval,
                             self.flat["actor"].data_ptr(), self.flat["critic"].data_ptr(),
                             self.flat["target_actor"].data_ptr(), self.flat["target_critic"].data_ptr(),
                             self.grads["actor"].data_ptr(), self.grads["critic"].data_ptr(),
                             self.exp_avg["actor"].data_ptr(), self.exp_avg_sq["actor"].data_ptr(),
                             self.exp_avg["critic"].data_ptr(), self.exp_avg_sq["critic"].data_ptr())
        self._h = c_void_p()
        if cfg.twin_critic:
            nv.check(self.lib.r2d2_learner_create_ex(byref(self._h), byref(c), byref(nv.LearnerOptions(1))))
        else:
            nv.check(self.lib.r2d2_learner_create(byref(self._h), byref(c)))
        self._rank = 0
        T, B, O, A, H, L = cfg.rows, cfg.batch, cfg.obs, cfg.act, cfg.hidden, cfg.learning
        dev = self.device
        # the batch has two slots (include/r2d2_b200.h): the attributes obs .. uniforms are views of the slot the NEXT
        # sample goes to; a plain caller never leaves slot 0
        self._slots = []
        for slot in (0, 1):
            b = nv.LearnerBuffers()
            nv.check(self.lib.r2d2_learner_buffers_get_slot(self._h, slot, byref(b)))
            self._slots.append({"obs": nv.view_f32(b.obs, (T, B, O), dev), "act": nv.view_f32(b.act, (T, B, A), dev),
                                "rew": nv.view_f32(b.rew, (T, B), dev), "term": nv.view_f32(b.term, (T, B), dev),
                                "states": nv.view_f32(b.states, (4, 2, B, H), dev),
                                "leaf_idx": nv.view_i64(b.leaf_idx, (B,), dev),
                                "uniforms": nv.view_f32(b.uniforms, (B,), dev)})
            w = c_void_p()
            nv.check(self.lib.r2d2_learner_is_weights(self._h, slot, byref(w)))
            self._slots[-1]["is_weight"] = nv.view_f32(w.value, (B,), dev)
        self._lib_slot = 0
        self._targets_ahead = False      # the fill slot's target chains already ran: its batch must not change any more
        self._bind_slot(0)
        # prioritized replay: the critic loss weights each sequence by the importance weight the draw wrote next to
        # its leaf index (DeviceReplay.sample_into); off, the library runs the unweighted TD kernels
        self.importance_weighting = cfg.is_exponent > 0
        nv.check(self.lib.r2d2_learner_set_importance_weighting(self._h, int(self.importance_weighting)))
        # optimiser step: Polyak target update fused into the Adam launches, per-net gradient-norm clipping before them
        nv.check(self.lib.r2d2_learner_set_target_tau(self._h, float(cfg.target_tau)))
        nv.check(self.lib.r2d2_learner_set_grad_clip(self._h, float(cfg.grad_clip_norm)))
        # n-step target and priorities: the library starts at the reference's; set only when asked for
        if not self.td_options.is_default:
            self.set_td_options(cfg.value_rescaling, cfg.rescaling_eps, cfg.priority_metric)
        gn = c_void_p()
        nv.check(self.lib.r2d2_learner_grad_norms(self._h, byref(gn)))
        self.grad_norms = nv.view_f32(gn.value, (2,), dev)   # [critic, actor] pre-clip norms of the last step
        self.q_value = nv.view_f32(b.q_value, (L * B, A), dev)
        self.target_q_value = nv.view_f32(b.target_q_value, (L * B, A), dev)
        self.td_sq = nv.view_f32(b.td_sq, (L * B,), dev)
        self.priority = nv.view_f32(b.priority, (B,), dev)
        self.losses = nv.view_f32(b.losses, (3 if cfg.twin_critic else 2,), dev)
        # TD3: critic 2's q (losses[2] is its loss) and the arena bytes the twin added; target noise only when asked for
        q2, off2, tb = c_void_p(), c_longlong(), nv.c_size_t()
        nv.check(self.lib.r2d2_learner_twin_buffers(self._h, byref(q2), byref(off2), byref(tb)))
        if int(off2.value) != self._critic2_off:
            raise nv.NativeError("critic 2 sits at float %d of the library's critic block, not %d"
                                 % (off2.value, self._critic2_off))
        self.q_value2 = nv.view_f32(q2.value, (L * B, A), dev) if cfg.twin_critic else None
        self.twin_added_bytes = int(tb.value)
        if cfg.target_noise > 0:
            self.set_target_smoothing()
        # learner metrics: the ring the library's metrics kernels write and its reader (None when off)
        self.metrics = metrics_mod.LearnerMetrics.attach(self) if cfg.metrics else None
        self.world = 1
        self._dist = None
        self._sync = None
        self._peer_buf = None
        self._peer_hdl = None
        self._sync_actor = None
        # global sampling: both batch slots move into one buffer per rank that every rank maps (here a plain one for a
        # single rank; enable_data_parallel replaces it by symmetric memory); off, the slots stay in the library's arena
        self._global_buf = self._global_hdl = None
        self.global_peer_ptrs = None
        # observation normalisation: the device statistics every attached replay shard's gathers read
        self.obs_norm = obs_norm_mod.ObsNormStats(cfg.obs, cfg.obs_norm_clip, self.device) if cfg.obs_norm else None
        if cfg.global_sampling:
            lay = self.global_layout(1)
            self.use_global_slots(torch.zeros(int(lay.bytes) // 4, dtype=torch.float32, device=self.device), lay)
            self.global_peer_ptrs = [self._global_buf.data_ptr()]

    def global_layout(self, world: int):
        """Bytes and offsets of one rank's global-sampling buffer (exchange block + two batch slots) at `world` ranks."""
        c = self.cfg
        lay = nv.GlobalLayout()
        nv.check(self.lib.r2d2_global_layout_for(c.rows, c.batch, c.obs, c.act, c.hidden, int(world), byref(lay)))
        return lay

    def use_global_slots(self, buf: torch.Tensor, lay):
        """Move both batch slots into `buf` (a zeroed float32 CUDA tensor of lay.bytes, laid out by global_layout): the
        replay shards of every rank store the drawn rows straight into them.  Only before the first step."""
        T, B, O, A, H = self.cfg.rows, self.cfg.batch, self.cfg.obs, self.cfg.act, self.cfg.hidden
        base, dev = buf.data_ptr(), self.device
        for slot in (0, 1):
            so = base + int(lay.slot_offset[slot])
            b = nv.LearnerBuffers()
            b.obs, b.act, b.rew, b.term = so + lay.off_obs, so + lay.off_act, so + lay.off_rew, so + lay.off_term
            b.states, b.leaf_idx, b.uniforms = so + lay.off_states, so + lay.off_leaf_idx, so + lay.off_uniforms
            nv.check(self.lib.r2d2_learner_set_slot_buffers(self._h, slot, byref(b), c_void_p(so + lay.off_is_weight)))
            self._slots[slot] = {"obs": nv.view_f32(b.obs, (T, B, O), dev), "act": nv.view_f32(b.act, (T, B, A), dev),
                                 "rew": nv.view_f32(b.rew, (T, B), dev), "term": nv.view_f32(b.term, (T, B), dev),
                                 "states": nv.view_f32(b.states, (4, 2, B, H), dev),
                                 "leaf_idx": nv.view_i64(b.leaf_idx, (B,), dev),
                                 "uniforms": nv.view_f32(b.uniforms, (B,), dev),
                                 "is_weight": nv.view_f32(so + lay.off_is_weight, (B,), dev),
                                 "shard": torch.as_tensor(nv._RawView(so + lay.off_shard, (B,), "<i4"), device=dev)}
            self._slots[slot]["is_weight"].fill_(1.0)
        self._global_buf = buf
        self._global_bytes = int(lay.bytes)
        self._bind_slot(self._fill_slot)

    def shard_of(self, leaf_idx: torch.Tensor) -> torch.Tensor:
        """The shard ids [B] (int32) next to a slot's leaf indices (global sampling)."""
        for s in self._slots:
            if "shard" in s and s["leaf_idx"].data_ptr() == leaf_idx.data_ptr():
                return s["shard"]
        raise nv.NativeError("global sampling writes back a batch slot's own leaf indices (engine.leaf_idx of the "
                             "trained batch); these are not a slot's")

    @property
    def td_options(self) -> td_options.TdOptions:
        c = self.cfg
        return td_options.TdOptions(c.value_rescaling, c.rescaling_eps, c.priority_metric)

    def set_td_options(self, value_rescaling: str, rescaling_eps: float, priority_metric: str):
        """Change the n-step target / priority options; allowed between any two steps (the TD kernel applies
        h_eps^-1 to the target critic's raw output, so nothing computed earlier depends on them)."""
        rescaling, eps, metric = td_options.TdOptions(value_rescaling, rescaling_eps, priority_metric).native()
        nv.check(self.lib.r2d2_learner_set_value_rescaling(self._h, rescaling, eps))
        nv.check(self.lib.r2d2_learner_set_priority_metric(self._h, metric))
        self.cfg.value_rescaling, self.cfg.rescaling_eps, self.cfg.priority_metric = value_rescaling, rescaling_eps, \
            priority_metric

    def set_target_smoothing(self, sigma: float | None = None, clip: float | None = None, seed: int | None = None,
                             rank: int | None = None):
        """TD3 target policy smoothing (sigma 0 = off); arguments left out keep the engine's setting.  The noise is a
        function of (seed, rank, iteration index, element): data-parallel ranks draw different noise, a resumed run the
        same as an uninterrupted one.  Refused while a prefetched batch's target chains have already run."""
        c = self.cfg
        sigma = c.target_noise if sigma is None else float(sigma)
        clip = c.target_noise_clip if clip is None else float(clip)
        seed = c.target_noise_seed if seed is None else int(seed)
        rank = self._rank if rank is None else int(rank)
        if not (0 <= seed < 2 ** 32 and 0 <= rank < 2 ** 32):
            raise ValueError("seed and rank are integers in [0, 2**32), got %r, %r" % (seed, rank))
        nv.check(self.lib.r2d2_learner_set_target_smoothing(self._h, sigma, clip, seed, rank))
        c.target_noise, c.target_noise_clip, c.target_noise_seed, self._rank = sigma, clip, seed, rank

    def _guard_fill(self):
        if self._targets_ahead:
            raise nv.NativeError("the engine's batch was filled by a step(prefetch=...) hook and its target chains "
                                 "have already run: call step(), or discard_prefetched(), before writing another batch")

    def discard_prefetched(self):
        """Drop a batch that a step(prefetch=...) hook drew ahead (its target chains are forgotten too): the next
        sample_into / set_batch starts a fresh sequence."""
        nv.check(self.lib.r2d2_learner_discard_prefetch(self._h, nv.current_stream()))
        self._targets_ahead = False

    def _bind_slot(self, slot: int):
        for k, v in self._slots[slot].items():
            setattr(self, k, v)
        self._fill_slot = slot

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            if getattr(self, "_peer_buf", None) is not None:
                # peers read this rank's gradient block until their last slice sum ran: completing the pending phase 3
                # (its wait kernel needs every peer's "slice delivered" flag) proves nobody touches the buffer any more
                try:
                    self.flush()
                    torch.cuda.synchronize(self.device)
                except Exception:
                    pass
            self._pending_finish = False
            self.lib.r2d2_learner_destroy(self._h)
            self._h = None
            self._peer_buf = self._peer_hdl = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- parameters -------------------------------------------------------------------------
    def views(self, net: str, what: str = "params"):
        self.flush()
        src = {"params": self.flat, "grads": self.grads, "exp_avg": self.exp_avg, "exp_avg_sq": self.exp_avg_sq}[what]
        return flat_views(self._block(src, net), self.cfg, "critic" in net)

    @property
    def nets(self) -> tuple:
        """The engine's nets: the reference's four, and critic 2 / target critic 2 with the twin critic."""
        return ("actor", "target_actor", "critic", "target_critic") + (
            ("critic2", "target_critic2") if self.cfg.twin_critic else ())

    def _block(self, src: dict, net: str) -> torch.Tensor:
        """A net's flat block in one of the buffer dicts: with the twin, "critic" / "target_critic" (and their moments
        and gradients) are the first half of the 2 P block, "critic2" / "target_critic2" the second."""
        if net.endswith("2"):
            if not self.cfg.twin_critic or net not in ("critic2", "target_critic2"):
                raise KeyError("%r: this engine has %s" % (net, ", ".join(self.nets)))
            return src[net[:-1]][self._critic2_off:self._critic2_off + self._n_critic]
        t = src[net]
        return t[:self._n_critic] if "critic" in net and self.cfg.twin_critic else t

    def state_dict(self, net: str):
        return OrderedDict((k, v.detach().clone()) for k, v in self.views(net).items())

    def load_state_dicts(self, actor, critic, target_actor=None, target_critic=None, critic2=None, target_critic2=None):
        """The reference's four nets (a target defaults to its net), and with the twin critic 2 and its target
        (target_critic2 defaults to critic2; left out, critic 2 keeps its weights).  actor / critic None: unchanged."""
        def put(net, sd):
            for k, v in self.views(net).items():
                v.copy_(torch.as_tensor(np.asarray(sd[k]) if not isinstance(sd[k], torch.Tensor) else sd[k],
                                        dtype=torch.float32).to(self.device))
        if actor is not None:
            put("actor", actor)
            put("target_actor", target_actor if target_actor is not None else actor)
        if critic is not None:
            put("critic", critic)
            put("target_critic", target_critic if target_critic is not None else critic)
        if critic2 is not None or target_critic2 is not None:
            if not self.cfg.twin_critic:
                raise ValueError("critic 2 weights given to an engine without the twin critic")
            if critic2 is not None:
                put("critic2", critic2)
            put("target_critic2", target_critic2 if target_critic2 is not None else critic2)

    def enable_data_parallel(self, require: bool | None = None):
        """Gradients are averaged over ranks at the two optimiser steps: by the library's own kernels over NVLink peer
        memory (`_attach_peers`, csrc/peer.cu), or - fallback / R2D2_DP_MODE=defer - by NCCL all-reduces of the flat
        buffers on a side stream.  `require` (default: WORLD_SIZE > 1 in the environment) turns a missing process group
        into an error instead of N silently independent learners."""
        import os
        import torch.distributed as dist
        from .dist_env import GradSync
        if require is None:
            require = int(os.environ.get("WORLD_SIZE", "1")) > 1
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            self._dist = dist
            self.world = dist.get_world_size()
            self._sync = GradSync(dist, self.world)
            self._sync_actor = GradSync(dist, self.world)
            self._rank = dist.get_rank()             # the target noise is keyed on (seed, rank): ranks draw their own
            if self.obs_norm is not None:
                self.obs_norm.dist = dist
            if self.cfg.target_noise > 0:
                self.set_target_smoothing()
            if self._dp_mode == "peer":
                self._attach_peers(dist)
            if self.cfg.global_sampling:
                self._attach_global_slots(dist)
            # both modes defer phase 3: the actor's weights are final only after it ran
            nv.check(self.lib.r2d2_learner_set_overlap_actor_inputs(self._h, 0))
            for net in ("actor", "critic", "target_actor", "target_critic"):
                dist.broadcast(self.flat[net], src=0)
            for d in (self.exp_avg, self.exp_avg_sq):
                for net in ("actor", "critic"):
                    dist.broadcast(d[net], src=0)
        elif require:
            raise nv.NativeError("WORLD_SIZE > 1 but torch.distributed is not initialised: call "
                                 "r2d2_b200.dist_env.DistEnv.from_environ().init_process_group() first "
                                 "(the drop-in learner.Learner does)")

    def _attach_peers(self, dist):
        """Move the gradient blocks into a buffer every rank of the node maps (torch symmetric memory: CUDA fabric /
        IPC handles exchanged through the process group's store) and hand the peer addresses to the library.  All ranks
        agree on the outcome; if any rank cannot map its peers, every rank falls back to the NCCL "defer" mode."""
        ok, why = 1, ""
        try:
            import torch.distributed._symmetric_memory as symm
            lay = nv.PeerLayout()
            nv.check(self.lib.r2d2_learner_peer_layout(self._h, self.world, byref(lay)))
            buf = symm.empty(int(lay.bytes) // 4, dtype=torch.float32, device=self.device)
            buf.zero_()
            hdl = symm.rendezvous(buf, dist.group.WORLD.group_name)
            ptrs = [int(p) for p in hdl.buffer_ptrs]
            if len(ptrs) != self.world or int(hdl.rank) != dist.get_rank() or ptrs[dist.get_rank()] != buf.data_ptr():
                raise RuntimeError("symmetric-memory handle does not match the process group")
        except Exception as e:  # noqa: BLE001 - any failure means "no peer mapping on this box"
            ok, why = 0, repr(e)[:200]
        agreed = torch.tensor([ok], dtype=torch.int32, device=self.device)
        dist.all_reduce(agreed, op=dist.ReduceOp.MIN)
        if int(agreed.item()) == 0:
            if dist.get_rank() == 0:
                print(f"[r2d2_b200] no peer-mapped gradient buffer ({why or 'another rank failed'}): "
                      "gradient exchange falls back to NCCL all-reduces (R2D2_DP_MODE=defer)", flush=True)
            self._dp_mode = "defer"
            return
        torch.cuda.synchronize(self.device)
        dist.barrier()                                   # every rank's flag words are zero before anyone signals
        arr = (c_void_p * self.world)(*ptrs)
        nv.check(self.lib.r2d2_learner_attach_peers(self._h, dist.get_rank(), self.world, arr))
        self._peer_buf, self._peer_hdl = buf, hdl
        na, nc = self.grads["actor"].numel(), self.grads["critic"].numel()
        oc, oa = int(lay.off_critic_grads) // 4, int(lay.off_actor_grads) // 4
        self.grads = {"actor": buf[oa:oa + na], "critic": buf[oc:oc + nc]}

    def _attach_global_slots(self, dist):
        """Global sampling: the batch slots and the exchange block in torch symmetric memory, one buffer per rank mapped
        by every rank of the node.  All ranks agree on the outcome (an all-reduce, as _attach_peers does) and raise
        together: there is no fallback, without peer mappings the option cannot run."""
        ok, why, buf, hdl, ptrs = 1, "", None, None, None
        lay = self.global_layout(self.world)
        try:
            import torch.distributed._symmetric_memory as symm
            buf = symm.empty(int(lay.bytes) // 4, dtype=torch.float32, device=self.device)
            buf.zero_()
            hdl = symm.rendezvous(buf, dist.group.WORLD.group_name)
            ptrs = [int(p) for p in hdl.buffer_ptrs]
            if len(ptrs) != self.world or ptrs[dist.get_rank()] != buf.data_ptr():
                raise RuntimeError("the symmetric-memory handle does not match the process group")
        except Exception as e:  # noqa: BLE001 - any failure on any rank stops every rank
            ok, why = 0, repr(e)[:200]
        agreed = torch.tensor([ok], dtype=torch.int32, device=self.device)
        dist.all_reduce(agreed, op=dist.ReduceOp.MIN)
        if int(agreed.item()) == 0:
            raise nv.NativeError("global sampling needs a buffer every rank maps (torch symmetric memory): "
                                 + (why or "another rank failed to set it up"))
        self.use_global_slots(buf, lay)
        torch.cuda.synchronize(self.device)
        dist.barrier()                                   # every rank's flag words are zero before anyone signals
        self._global_hdl = hdl
        self.global_peer_ptrs = ptrs

    def peer_status(self) -> int:
        """0, or 1 when a bounded wait for a peer's flag expired inside the gradient-exchange kernels."""
        if self._peer_buf is None:
            return 0
        st = c_int(0)
        nv.check(self.lib.r2d2_learner_peer_status(self._h, byref(st), nv.current_stream()))
        return int(st.value)

    def replicas_identical(self) -> bool:
        """Data-parallel invariant: parameters and Adam moments are bit-identical on every rank."""
        if self._dist is None:
            return True
        self.flush()
        if self.peer_status() != 0:
            return False
        ts = [self.flat[n] for n in ("actor", "critic", "target_actor", "target_critic")]
        ts += [d[n] for d in (self.exp_avg, self.exp_avg_sq) for n in ("actor", "critic")]
        return self._sync.replicas_identical(ts)

    # ---- batch ------------------------------------------------------------------------------
    def set_batch(self, batch: dict):
        """Copy an already sampled time-major batch (replay_memory.py:123-136 layout) into the engine.  An optional
        batch["is_weight"] [B] holds the importance weights; without it every weight is 1."""
        cv = lambda x: torch.as_tensor(np.asarray(x) if not isinstance(x, torch.Tensor) else x,  # noqa: E731
                                       dtype=torch.float32).to(self.device, non_blocking=True)
        self._guard_fill()
        self.obs.copy_(cv(batch["obs"]))
        self.act.copy_(cv(batch["act"]))
        self.rew.copy_(cv(batch["rew"]).reshape(self.rew.shape))
        self.term.copy_(cv(batch["term"]).reshape(self.term.shape))
        for i, k in enumerate(("a_state", "ta_state", "c_state", "tc_state")):
            self.states[i].copy_(cv(batch[k]))
        if "is_weight" in batch:
            self.is_weight.copy_(cv(batch["is_weight"]).reshape(self.is_weight.shape))
        elif self.importance_weighting:
            self.is_weight.fill_(1.0)

    # ---- one learner iteration (learner.py:86-132) on the batch currently in the engine ------------
    def step(self, prefetch=None):
        """One learner iteration on the batch in the engine (learner.py:86-132).

        `prefetch(engine, used)`, if given, is called exactly once per step and must (1) write back the priorities of
        the batch this step trained on - `used.leaf_idx`, `used.priority` - and (2) fill the engine's batch buffers
        (`obs .. states`, e.g. `DeviceReplay.sample_into`) with the NEXT batch.  It is called as early as the data flow
        allows - right after the critic phase, when the priorities exist - and the next batch's target chains run
        straight away, in the middle of this iteration: they read only the target nets, so they are the independent
        work that lets the data-parallel ranks drift by a millisecond or two without waiting for each other (and on
        one GPU the input projections hide under their scans as before).  On iterations that update the target nets
        (hard copy, or the Polyak blend of `target_tau` < 1, which starts at the critic's optimiser step) it is called at
        the end of the step instead, and a deferred data-parallel phase 3 is completed before the next critic phase.
        At `target_interval` 1 that is every iteration: the next batch's target chains never run ahead.  On one GPU the
        critic BPTT (and the twin's chain) may still run on the library's second stream while the hook runs: the hook
        may read `used.priority` and `used.losses[0]`, the rest of `used.losses` is complete when step() returns.

        Data parallel, mode "peer" (default): the gradient blocks are summed by the library's own kernels over NVLink
        peer memory inside the phases (csrc/peer.cuh); the actor's optimiser step of iteration i runs after the critic
        phase of iteration i+1.  Mode "defer" (fallback): NCCL all-reduces on a side stream, the actor's waited for
        after the next critic phase; the hook then runs at the end of the step."""
        s = nv.current_stream()
        scale = 1.0 / self.world
        if self._fill_slot != self._lib_slot:
            nv.check(self.lib.r2d2_learner_select_batch(self._h, self._fill_slot))
            self._lib_slot = self._fill_slot
        self._targets_ahead = False
        if self._pending_finish and self._finish_updates_targets():
            self.flush()                                                  # the target chains below read the target nets
        nv.check(self.lib.r2d2_learner_critic_phase(self._h, s))
        if self._dist is not None and self._dp_mode == "defer":
            self._sync.start(self.grads["critic"])                       # side stream
            self.flush()                                                  # phase 3 of the previous iteration (actor Adam)
            nv.check(self.lib.r2d2_learner_actor_forward(self._h, s))    # reads no critic weights: overlaps the all-reduce
            self._sync.wait(self.device)
            nv.check(self.lib.r2d2_learner_actor_phase(self._h, scale, s))
            self._sync_actor.start(self.grads["actor"])
            self._pending_finish = True
            if prefetch is not None:
                self._run_prefetch(prefetch)
            return
        self.flush()                                                      # phase 3 of the previous iteration, if deferred
        ahead = prefetch is not None and not self._finish_updates_targets()
        if ahead:
            self._run_prefetch(prefetch)
            nv.check(self.lib.r2d2_learner_target_phase(self._h, self._fill_slot, s))
            self._targets_ahead = True
        nv.check(self.lib.r2d2_learner_actor_forward(self._h, s))
        nv.check(self.lib.r2d2_learner_actor_phase(self._h, scale, s))
        if self._dist is not None:   # "peer": signal / slice-sum / wait kernels are issued by the phases themselves
            self._pending_finish = True
        else:
            nv.check(self.lib.r2d2_learner_finish_phase(self._h, scale, s))
        if prefetch is not None and not ahead:
            self._run_prefetch(prefetch)

    def _run_prefetch(self, prefetch):
        from types import SimpleNamespace
        used = SimpleNamespace(leaf_idx=self.leaf_idx, priority=self.priority, losses=self.losses,
                               is_weight=self.is_weight)
        self._bind_slot(1 - self._fill_slot)     # the phases still in flight keep reading the other slot
        prefetch(self, used)

    def _finish_updates_targets(self) -> bool:
        k = self.cfg.target_interval
        return k > 0 and (int(self.lib.r2d2_learner_step_count(self._h)) + 1) % k == 0

    def flush(self):
        """Complete a deferred phase 3 (actor all-reduce wait + Adam + step counter + target update)."""
        if self._pending_finish:
            if self._dp_mode != "peer":
                self._sync_actor.wait(self.device)
            nv.check(self.lib.r2d2_learner_finish_phase(self._h, 1.0 / self.world, nv.current_stream()))
            self._pending_finish = False

    @property
    def step_count(self) -> int:
        self.flush()
        return int(self.lib.r2d2_learner_step_count(self._h))

    # ---- full training state (SURVEY 8f N3: the reference checkpoints weights only and cannot resume) ---------------
    def training_state(self) -> dict:
        """Everything a restart needs: the four nets (reference keys), both Adam moment sets, the step counter, and the
        n-step target / priority options the critic was trained under."""
        torch.cuda.synchronize(self.device)
        out = {net: self.state_dict(net) for net in self.nets}
        for net in [n for n in self.nets if not n.startswith("target")]:
            out[net + "_optimizer"] = {"exp_avg": OrderedDict((k, v.detach().clone()) for k, v in self.views(net, "exp_avg").items()),
                                       "exp_avg_sq": OrderedDict((k, v.detach().clone()) for k, v in self.views(net, "exp_avg_sq").items())}
        out["step"] = self.step_count
        o = self.td_options
        out.update(value_rescaling=o.value_rescaling, rescaling_eps=float(o.rescaling_eps), priority_metric=o.priority_metric)
        c = self.cfg
        out.update(twin_critic=bool(c.twin_critic), target_noise=float(c.target_noise),
                   target_noise_clip=float(c.target_noise_clip), target_noise_seed=int(c.target_noise_seed))
        if getattr(self, "obs_norm", None) is not None:
            out["obs_norm"] = self.obs_norm.state()
        return out

    def load_training_state(self, st: dict):
        """Refuses a state saved under other target / priority options: a critic trained in one value space means nothing
        in the other.  A state without them was saved by a build that had only the reference's (reference, squared).
        Likewise a twin-critic state and a single-critic engine, or the other way round (a state without the key is
        single-critic).  The target-noise settings of the state are informational: the engine keeps its own.  Observation
        normalisation on one side and off on the other is refused too, and so is another clip; otherwise the statistics
        are restored."""
        stats = getattr(self, "obs_norm", None)
        saved_norm = bool((st.get("obs_norm") or {}).get("enabled", False))
        if saved_norm != (stats is not None):
            raise ValueError("training state was saved with obs_norm=%r; this engine runs obs_norm=%r: nets trained on "
                             "normalised observations mean nothing on raw ones, and the other way round"
                             % (saved_norm, stats is not None))
        if stats is not None and np.float32(st["obs_norm"]["clip"]) != np.float32(stats.clip):
            raise ValueError("training state was saved with obs_norm_clip=%r; this engine runs obs_norm_clip=%r: the nets "
                             "were trained on differently clamped observations" % (st["obs_norm"]["clip"], stats.clip))
        saved_twin = bool(st.get("twin_critic", False))
        if saved_twin != bool(self.cfg.twin_critic):
            raise ValueError("training state was saved with twin_critic=%r; this engine runs twin_critic=%r"
                             % (saved_twin, bool(self.cfg.twin_critic)))
        def key(o):
            return (o.value_rescaling, float(np.float32(o.rescaling_eps)) if o.value_rescaling == "invertible" else None,
                    o.priority_metric)
        saved = td_options.TdOptions(st.get("value_rescaling", "reference"),
                                     st.get("rescaling_eps", td_options.DEFAULT_EPS), st.get("priority_metric", "squared"))
        mine = self.td_options
        if key(saved) != key(mine):
            raise ValueError("training state was saved with value_rescaling=%r rescaling_eps=%r priority_metric=%r; this "
                             "engine runs value_rescaling=%r rescaling_eps=%r priority_metric=%r"
                             % (saved.value_rescaling, saved.rescaling_eps, saved.priority_metric, mine.value_rescaling,
                                mine.rescaling_eps, mine.priority_metric))
        self.load_state_dicts(st["actor"], st["critic"], st.get("target_actor"), st.get("target_critic"),
                              st.get("critic2"), st.get("target_critic2"))
        for net in [n for n in self.nets if not n.startswith("target")]:
            opt = st.get(net + "_optimizer")
            if opt is not None:
                for what in ("exp_avg", "exp_avg_sq"):
                    for k, v in self.views(net, what).items():
                        v.copy_(torch.as_tensor(opt[what][k], dtype=torch.float32).to(self.device))
        nv.check(self.lib.r2d2_learner_set_step_count(self._h, int(st.get("step", 0))))
        if getattr(self, "metrics", None) is not None:
            self.metrics.next = int(st.get("step", 0))    # the ring's numbering continues from the resumed step
        if stats is not None:
            stats.load_state(st["obs_norm"])

    @property
    def launches_per_iteration(self) -> int:
        return int(self.lib.r2d2_learner_launches_per_iteration(self._h))


class DeviceReplay:
    """One replay shard in HBM with a 32-ary sum tree (one leaf per stored row)."""

    def __init__(self, cfg: PathConfig, capacity_rows: int, max_sequences: int = 0, device=None):
        if not torch.cuda.is_available():
            raise nv.NativeError("DeviceReplay needs a CUDA device; there is no CPU fallback")
        self.lib = nv.lib()
        self.cfg = cfg
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        torch.cuda.set_device(self.device)
        rc = nv.ReplayConfig(cfg.obs, cfg.act, cfg.hidden, cfg.burn_in, cfg.learning, cfg.n_step,
                             int(capacity_rows), int(max_sequences))
        self._h = c_void_p()
        opt = nv.ReplayOptions(REPLAY_STATE_DTYPES[cfg.replay_state_dtype], REPLAY_STATE_MEMORY[cfg.replay_state_memory])
        nv.check(self.lib.r2d2_replay_create_ex(byref(self._h), byref(rc), byref(opt)))
        if cfg.priority_exponent != 1.0:   # leaves hold p^alpha; actors and write-backs keep passing raw priorities
            nv.check(self.lib.r2d2_replay_set_priority_exponent(self._h, float(cfg.priority_exponent)))
        self._group = None                 # the engine whose rank / world / buffers global sampling uses
        self._obs_norm = None              # the ObsNormStats the gathers read (attach_obs_norm)

    def attach_group(self, eng: LearnerEngine):
        """Global sampling: this shard becomes rank eng's shard of the group of eng.world ranks; from then on
        sample_into draws the rank's B sequences of one W*B global batch from all shards, and update_priorities writes
        the trained batch's priorities back into the shards that own its rows (a collective: every rank calls both, in
        the same order).  The engine needs PathConfig.global_sampling."""
        if not eng.cfg.global_sampling or eng.global_peer_ptrs is None:
            raise nv.NativeError("attach_group needs an engine with PathConfig.global_sampling")
        ec, rc = eng.cfg, self.cfg
        if (ec.obs, ec.act, ec.hidden, ec.rows) != (rc.obs, rc.act, rc.hidden, rc.rows):
            raise nv.NativeError("replay shard (obs %d act %d hidden %d rows %d) does not match the engine (obs %d act %d "
                                 "hidden %d rows %d)" % (rc.obs, rc.act, rc.hidden, rc.rows, ec.obs, ec.act, ec.hidden, ec.rows))
        arr = (c_void_p * eng.world)(*eng.global_peer_ptrs)
        nv.check(self.lib.r2d2_replay_attach_group(self._h, eng._rank, eng.world, ec.batch, arr, eng._global_bytes))
        self._group = eng

    def attach_obs_norm(self, stats):
        """Every gather of this shard (sample_into, the global draw, r2d2_replay_gather) normalises the batch's obs with
        the fp32 pair of `stats` (an ObsNormStats, e.g. LearnerEngine.obs_norm), read at each gather; None detaches."""
        if stats is None:
            nv.check(self.lib.r2d2_replay_set_obs_normalizer(self._h, None, None, 0.0))
        else:
            if stats.O != self.cfg.obs:
                raise nv.NativeError("obs normaliser of width %d for a shard of obs %d" % (stats.O, self.cfg.obs))
            nv.check(self.lib.r2d2_replay_set_obs_normalizer(self._h, nv.dptr(stats.mean_f), nv.dptr(stats.inv_std_f),
                                                             float(stats.clip)))
        self._obs_norm = stats

    @property
    def group(self):
        """The engine this shard samples globally for (attach_group), or None."""
        return self._group

    def global_draw(self, eng: LearnerEngine, stage: int = -1, generator: torch.Generator | None = None,
                    u: torch.Tensor | None = None, beta: float | None = None):
        """Global sampling's draw into the engine's fill slot (what sample_into does once attached).  stage 0 writes
        this rank's uniforms and publishes them with the shard root, 1 draws, gathers and signals delivery, 2 waits for
        every owner and forms the weights; -1 runs all three.  In-process groups issue each stage for every rank before
        the next, so that no wait spins."""
        if self._group is None or eng is not self._group:
            raise nv.NativeError("this shard draws globally only for the engine it was attached to")
        eng._guard_fill()
        if stage in (0, -1):
            if u is None:
                eng.uniforms.copy_(torch.rand(eng.cfg.batch, device=self.device, generator=generator))
            else:
                eng.uniforms.copy_(u)
        b = eng.cfg.is_exponent if beta is None else float(beta)
        if not 0.0 <= b <= 1.0:
            raise ValueError("beta must lie in [0, 1], got %r" % (b,))
        nv.check(self.lib.r2d2_replay_global_draw(self._h, int(stage), eng._fill_slot, int(eng.importance_weighting), b,
                                                  nv.current_stream()))

    def global_write_back(self, leaf_idx: torch.Tensor, prio: torch.Tensor, stage: int = -1):
        """Global sampling's write-back of the trained batch (what update_priorities does once attached): leaf_idx is
        that slot's engine.leaf_idx.  stage 0 publishes this rank's records, 1 waits for all and applies this shard's;
        -1 runs both."""
        shard = self._group.shard_of(leaf_idx)
        nv.check(self.lib.r2d2_replay_global_write_back(self._h, int(stage), nv.dptr(leaf_idx, torch.int64),
                                                        nv.dptr(shard, torch.int32), nv.dptr(prio),
                                                        nv.current_stream()))

    def global_status(self) -> int:
        """0, or 1 when a bounded wait of the global-sampling kernels expired."""
        if self._group is None:
            return 0
        st = c_int(0)
        nv.check(self.lib.r2d2_replay_global_status(self._h, byref(st), nv.current_stream()))
        return int(st.value)

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            self.lib.r2d2_replay_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def add_episode(self, obs, act, rew, term, states, priority):
        """obs [n_rows,O], act [n_rows,A], rew/term [n_rows], states [n_real,4,2,H], priority [n_starts] (host)."""
        obs, po = nv.host_f32(obs)
        act, pa = nv.host_f32(act)
        rew, pr = nv.host_f32(np.asarray(rew).reshape(-1))
        term, pt = nv.host_f32(np.asarray(term).reshape(-1))
        states, ps = nv.host_f32(states)
        priority, pp = nv.host_f32(np.asarray(priority).reshape(-1))
        nv.check(self.lib.r2d2_replay_add_episode(self._h, po, pa, pr, pt, ps, obs.shape[0], states.shape[0], pp,
                                                  priority.shape[0], nv.current_stream()))

    def add_episodes(self, episodes, obs_norm=None):
        """One actor file in one native call (LearnerReplayMemory.load, replay_memory.py:138-157).  `episodes`: list of
        (obs [n,O], act [n,A], rew [n], term [n], states [n_real,4,2,H], priority [n_starts]) host arrays.  Returns
        (row_start per episode, episodes evicted by the call, sequence counter).  `obs_norm` (an ObsNormStats): the
        call's observation moments (r2d2_replay_add_episodes_ex) are merged into its pending block."""
        if not episodes:
            return [], 0, None
        n_rows = np.asarray([e[0].shape[0] for e in episodes], np.int32)
        n_starts = np.asarray([len(e[5]) for e in episodes], np.int32)
        R, H = int(n_rows.sum()), self.cfg.hidden
        obs = np.concatenate([np.asarray(e[0], np.float32) for e in episodes])
        act = np.concatenate([np.asarray(e[1], np.float32) for e in episodes])
        rew = np.concatenate([np.asarray(e[2], np.float32).reshape(-1) for e in episodes])
        term = np.concatenate([np.asarray(e[3], np.float32).reshape(-1) for e in episodes])
        states = np.zeros((R, 4, 2, H), np.float32)
        leaf = np.zeros(R, np.float32)
        off = 0
        for e, n in zip(episodes, n_rows):
            st = np.asarray(e[4], np.float32)
            if st.shape[1:] != (4, 2, H) or st.shape[0] > n:
                raise ValueError("recurrent states %r do not fit an episode of %d rows at hidden %d" % (st.shape, n, H))
            states[off:off + st.shape[0]] = st
            leaf[off:off + len(e[5])] = np.asarray(e[5], np.float32).reshape(-1)
            off += int(n)
        if obs.shape != (R, self.cfg.obs) or act.shape != (R, self.cfg.act):
            raise ValueError("episode rows %r / %r do not match the shard (obs %d, act %d)" % (obs.shape, act.shape,
                                                                                           self.cfg.obs, self.cfg.act))
        starts = np.zeros(len(episodes), np.int64)
        n_evicted, counter = c_longlong(0), c_longlong(0)
        P = lambda a: a.ctypes.data_as(c_void_p)  # noqa: E731
        if obs_norm is None:
            nv.check(self.lib.r2d2_replay_add_episodes(self._h, len(episodes), P(n_rows), P(n_starts), P(obs), P(act),
                                                       P(rew), P(term), P(states), P(leaf), P(starts), byref(n_evicted),
                                                       byref(counter), nv.current_stream()))
        else:
            bad = c_longlong(0)
            nv.check(self.lib.r2d2_replay_add_episodes_ex(self._h, len(episodes), P(n_rows), P(n_starts), P(obs), P(act),
                                                          P(rew), P(term), P(states), P(leaf), P(starts), byref(n_evicted),
                                                          byref(counter), nv.dptr(obs_norm.ingest_block, torch.float64),
                                                          byref(bad), nv.current_stream()))
            obs_norm.add_ingest(int(bad.value))
        return starts.tolist(), int(n_evicted.value), int(counter.value)

    def sample_indices(self, u: torch.Tensor) -> torch.Tensor:
        leaf = torch.empty(u.numel(), dtype=torch.int64, device=self.device)
        nv.check(self.lib.r2d2_replay_sample(self._h, nv.dptr(u), u.numel(), nv.dptr(leaf, torch.int64), None, None,
                                             None, None, None, nv.current_stream()))
        return leaf

    def sample_into(self, eng: LearnerEngine, generator: torch.Generator | None = None, u: torch.Tensor | None = None,
                    beta: float | None = None):
        """Draw eng.cfg.batch starts and gather the time-major batch straight into the engine's buffers.  With the
        engine's importance weighting on, the draw also writes eng.is_weight with exponent `beta` (default
        eng.cfg.is_exponent; pass it per draw to anneal it)."""
        ec, rc = eng.cfg, self.cfg
        eng._guard_fill()
        if (ec.obs, ec.act, ec.hidden, ec.rows) != (rc.obs, rc.act, rc.hidden, rc.rows):
            raise nv.NativeError("replay shard (obs %d act %d hidden %d rows %d) does not match the engine (obs %d act %d "
                                 "hidden %d rows %d)" % (rc.obs, rc.act, rc.hidden, rc.rows, ec.obs, ec.act, ec.hidden, ec.rows))
        if self._group is not None:
            self.global_draw(eng, -1, generator=generator, u=u, beta=beta)
            return
        if u is None:
            eng.uniforms.copy_(torch.rand(eng.cfg.batch, device=self.device, generator=generator))
        else:
            eng.uniforms.copy_(u)
        if eng.importance_weighting:
            b = ec.is_exponent if beta is None else float(beta)
            if not 0.0 <= b <= 1.0:
                raise ValueError("beta must lie in [0, 1], got %r" % (b,))
            nv.check(self.lib.r2d2_replay_sample_weighted(self._h, nv.dptr(eng.uniforms), eng.cfg.batch, b,
                                                          nv.dptr(eng.leaf_idx, torch.int64), nv.dptr(eng.is_weight),
                                                          nv.dptr(eng.obs), nv.dptr(eng.act), nv.dptr(eng.rew),
                                                          nv.dptr(eng.term), nv.dptr(eng.states), nv.current_stream()))
            return
        nv.check(self.lib.r2d2_replay_sample(self._h, nv.dptr(eng.uniforms), eng.cfg.batch,
                                             nv.dptr(eng.leaf_idx, torch.int64), nv.dptr(eng.obs), nv.dptr(eng.act),
                                             nv.dptr(eng.rew), nv.dptr(eng.term), nv.dptr(eng.states),
                                             nv.current_stream()))

    def update_priorities(self, leaf_idx: torch.Tensor, prio: torch.Tensor):
        """Write raw priorities back; the leaves store prio^alpha (PathConfig.priority_exponent).  Global sampling:
        leaf_idx must be the trained slot's (engine.leaf_idx); every rank's records reach the shards that own them."""
        if self._group is not None:
            self.global_write_back(leaf_idx, prio)
            return
        nv.check(self.lib.r2d2_replay_update_priorities(self._h, nv.dptr(leaf_idx, torch.int64), nv.dptr(prio),
                                                        leaf_idx.numel(), nv.current_stream()))

    def device_bytes(self) -> int:
        """Bytes of device memory the shard holds: rows, tree, and the ingest / restore staging block once used (not the
        states of replay_state_memory="host")."""
        n = c_size_t(0)
        nv.check(self.lib.r2d2_replay_device_bytes(self._h, byref(n)))
        return int(n.value)

    def host_bytes(self) -> int:
        """Bytes of pinned host memory the shard holds: the recurrent states under replay_state_memory="host", else 0."""
        n = c_size_t(0)
        nv.check(self.lib.r2d2_replay_host_bytes(self._h, byref(n)))
        return int(n.value)

    def stats(self) -> dict:
        st = nv.ReplayStats()
        nv.check(self.lib.r2d2_replay_stats(self._h, byref(st), nv.current_stream()))
        return {k: getattr(st, k) for k, _ in nv.ReplayStats._fields_}

    def decode(self, leaf_idx):
        leaf = np.ascontiguousarray(np.asarray(leaf_idx.cpu() if isinstance(leaf_idx, torch.Tensor) else leaf_idx),
                                    dtype=np.int64)
        ep = np.empty_like(leaf)
        sq = np.empty_like(leaf)
        nv.check(self.lib.r2d2_replay_decode(self._h, leaf.ctypes.data_as(c_void_p), leaf.size,
                                             ep.ctypes.data_as(c_void_p), sq.ctypes.data_as(c_void_p)))
        return ep, sq

    def tree_level(self, level: int) -> torch.Tensor:
        p, n = c_void_p(), c_longlong()
        nv.check(self.lib.r2d2_replay_tree_level(self._h, level, byref(p), byref(n)))
        return nv.view_f32(p.value, (n.value,), self.device)

    # ---- snapshots (r2d2_b200.replay_snapshot holds the file format) -------------------------------------------------
    def snapshot_info(self) -> dict:
        """The shard's sizes, alpha, state storage, capacity and counters (what a snapshot's header records)."""
        info = nv.ReplaySnapshotInfo()
        nv.check(self.lib.r2d2_replay_export_info(self._h, byref(info)))
        return {k: getattr(info, k) for k, _ in nv.ReplaySnapshotInfo._fields_}

    def episodes(self):
        """The live episodes in FIFO order: (row_start, n_rows, n_starts, serial) int64 arrays."""
        E = int(self.snapshot_info()["n_episodes"])
        rs, nr, ns, se = (np.zeros(E, np.int64), np.zeros(E, np.int32), np.zeros(E, np.int32), np.zeros(E, np.int64))
        P = lambda a: a.ctypes.data_as(c_void_p)  # noqa: E731
        nv.check(self.lib.r2d2_replay_export_episodes(self._h, P(rs), P(nr), P(ns), P(se)))
        return rs, nr.astype(np.int64), ns.astype(np.int64), se

    def save_snapshot(self, path, world: int = 1, rank: int = 0, learner_step: int = 0, **kw):
        """Write the shard, with the device's CUDA RNG state, to one file (replay_snapshot.save).  The stream is idle
        afterwards; the shard is unchanged."""
        from . import replay_snapshot
        return replay_snapshot.save(self, path, world=world, rank=rank, learner_step=learner_step, **kw)

    def load_snapshot(self, path, world: int | None = None, restore_rng: bool = True, **kw) -> dict:
        """Restore a snapshot into this EMPTY shard (replay_snapshot.load): the same capacity gives back every row, leaf
        and tree level; another capacity compacts the episodes from row 0 and drops the oldest that do not fit.  A
        different state storage is converted.  Refused (the shard stays or is left empty) for other sizes, another
        alpha, another world size when `world` is given, a truncated file, a bad leaf or an fp16 overflow."""
        from . import replay_snapshot
        return replay_snapshot.load(self, path, world=world, restore_rng=restore_rng, **kw)

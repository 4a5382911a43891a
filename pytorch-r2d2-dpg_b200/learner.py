"""Drop-in for the reference's learner.py: `Learner(n_actors)`, `.run()`, `.save_model()`,
`.update_target_model()`, `learner_process(n_actors)` (learner.py:18-67) with the same attributes,
hyper-parameter literals, cwd-relative ./model_data and ./memory_data protocol and checkpoint keys -
so the reference's r2d2.py launcher runs unchanged - while every iteration of the loop body
(learner.py:84-139) executes in libr2d2_b200 (hand-written sm_90a CUDA):

    memory.sample()          -> DeviceReplay.sample_into   (sum-tree draw + gather kernels, HBM resident)
    burn-in / unrolls / BPTT -> LearnerEngine.step         (persistent cluster LSTM scans + tensor-core GEMMs)
    target, loss, priorities -> fused TD/priority kernel, written back into the sum tree on device

Data-parallel form (SURVEY 8e): launch `learner_process` once per GPU under torchrun (RANK / LOCAL_RANK /
WORLD_SIZE in the environment).  `Learner.__init__` then binds cuda:LOCAL_RANK, joins the NCCL process group,
ingests only the actors i with i mod WORLD_SIZE == RANK into its own HBM replay shard, and the two flat
gradient blocks are summed over the ranks by the library's peer-memory kernels inside the iteration (csrc/peer.cu);
rank 0 alone writes model.pt.  Nothing else crosses GPUs.

Prioritized replay (R2D2's, absent from the reference): R2D2_PRIORITY_EXPONENT (alpha, default 1) and R2D2_IS_EXPONENT
(beta, default 0) in the environment.  The defaults are the reference's behaviour; published R2D2 uses 0.9 / 0.6.
Under data parallelism each rank normalises the weights over its own batch, and draws from its own shard - unless
R2D2_GLOBAL_SAMPLING=1 (default 0): then the ranks draw one global batch of WORLD_SIZE * batch sequences from the union
of the shards in proportion to p^alpha, as the reference's single replay does, every rank trains on its B of them and the
weights are normalised over the global batch (the kernels of csrc/global_replay.cu and csrc/replay.cu, in the learner's
stream; the batch slots live in torch symmetric memory).  A host barrier follows every ingest in that mode.

Optimiser step: R2D2_TARGET_TAU (Polyak weight tau of the target update, default 1 = the reference's hard copy),
R2D2_TARGET_INTERVAL (iterations between target updates, default 500 = the reference's target_update_inverval; DDPG-style
soft updates use tau 0.005 at interval 1) and R2D2_GRAD_CLIP (global gradient-norm bound per net, default 0 = off).

n-step target and priorities (r2d2_b200.td_options, read the same way by the drop-in Actor and ActorPool):
R2D2_VALUE_RESCALING=reference|invertible (default reference: the reference's y = h(R + gamma^n (1-d) Q') with
h(x) = sign(x)(sqrt(|x|+1) - 1), no eps x and no inverse on the bootstrap; invertible: published R2D2's
y = h_eps(R + gamma^n (1-d) h_eps^-1(Q')), h_eps = h + eps x), R2D2_RESCALING_EPS (eps, default 1e-3) and
R2D2_PRIORITY_METRIC=squared|abs (default squared: the reference's eta max + (1-eta) mean of squared TD errors; abs: of
absolute ones, R2D2's).  Any other value raises.  The checkpoint records them and a resume under other settings is refused.

TD3's target (r2d2_b200.td3_options): R2D2_TWIN_CRITIC=0|1 (default 0; 1 adds a second critic and target critic and
bootstraps from the minimum of the two), R2D2_TARGET_NOISE (target policy smoothing sigma, default 0 = off),
R2D2_TARGET_NOISE_CLIP (default 0.5) and R2D2_TARGET_NOISE_SEED (default 0).  model.pt keeps its four reference keys
(critic 1 is the reference's critic); the resumable checkpoint holds critic 2 as well, and a resume across a twin /
single-critic change is refused.

Replay storage: R2D2_REPLAY_STATE_DTYPE=float32|float16 (default float32).  float16 keeps the four nets' stored (h, c) of
every replay row in fp16 - nearly twice the rows in the same HBM (the ring is capped at 60 % of free HBM) - rounded once
at ingest; an actor file holding a finite state of magnitude >= 65520 is refused whole.  Any other value raises.  The
setting may change across a resume: a replay snapshot in the other type is converted when it is restored.
R2D2_REPLAY_HOST_GB (default 0: the states stay in HBM) is the pinned host memory, in GB per rank, a replay shard may
use for those states: above 0 every row's (h, c) lives in mapped, page-locked host memory and only obs, act, reward,
terminal and the sum tree take HBM (1,585 bytes per row at obs 376, act 17), so the reference's 5 M sequences fit one
GPU.  The ring is then the least of the wanted rows, 60 % of the free HBM and the rows this budget holds (16 H bytes
per row in float16, 32 H in float32); the learner prints which applies.  The gather reads each drawn sequence's start
states over the host link and the batch is bit-identical.  A negative, non-finite or non-numeric value raises.  It may
change across a resume: snapshots do not depend on where the states live.

Replay snapshots: R2D2_REPLAY_SNAPSHOT_INTERVAL (learner steps between snapshots, default 0 = never; a multiple of
memory_update_interval, 50, else it raises).  After the ingest of every such step the learner writes
./model_data/replay_snapshot/step{N}/: learner_state.pt (the training state at step N, so the weights and the replay
belong to the same step), one shard{rank}of{world} per rank (r2d2_b200.replay_snapshot: the HBM shard, its sum-tree
leaves, its bookkeeping and the CUDA RNG state that draws the next batch) and, once every rank has written, a COMPLETE
marker from rank 0; the older snapshot directories are then deleted, so at most two are ever on disk.  The loop stalls
while a snapshot is written.  With R2D2_RESUME=1 and a complete snapshot present, the learner resumes from the newest
one - its training state (not the top-level learner_state.pt, which may be newer), its own shard and the RNG state -
so that the run continues bit for bit as if it had not stopped, and the warm-up gate passes at once when the restored
shard holds enough sequences.  A snapshot written at another world size is refused (re-sharding is not supported).
Without a complete snapshot the resume loads learner_state.pt alone and the replay starts empty, as before.  Actor files
not yet ingested stay on disk and are ingested after the resume as usual.

Observation normalisation (r2d2_b200.obs_norm): R2D2_OBS_NORM=0|1 (default 0) and R2D2_OBS_NORM_CLIP (default 5; finite
and > 0, else it raises).  On, the learner keeps float64 running mean / variance statistics of every observation row it
ingests (not the actors' n_step pad rows, nor rows holding NaN or +-inf), and every net reads
clamp((obs - mean) / std, -clip, clip) in place of the raw observation: the replay gather writes it into the batch, and
model.pt gains an `obs_norm` entry {mean_f, inv_std_f, clip} (next to its four reference keys, once a row was seen)
from which the drop-in Actor and ActorPool normalise what they act on.  The replay and its snapshots keep raw rows.  The
statistics change only right after the loop's ingests (and once before the first step), merged over the data-parallel
ranks in rank order, so every rank holds the same bits.  The checkpoint records them; a resume across an on / off
change, or across another clip, is refused.

Learner metrics (r2d2_b200.metrics): R2D2_METRICS=0|1 (default 0; any other value raises).  On, the library reduces one
record per iteration on the device (losses, Q / target / |TD error| / priority / importance-weight statistics, actor
saturation, both gradient norms, non-finite count; include/r2d2_b200.h), and at every log point (every 100 steps) and
when run() returns each rank appends the iterations finished since its last read to
./model_data/metrics/learner_rank{r}.csv (a header row when the file is new, then one row per iteration); rank 0 prints
one summary line of the interval's means after `learning step: N`.  No collective is added: each rank logs its own
batch, and the gradient norms, taken of the rank mean, are the same on every rank.  Training is bit-identical either way.
"""
import math
import os
import re
import shutil
from time import sleep, time

import numpy as np
import torch

from replay_memory import LearnerReplayMemory
from utils import get_obs

WALKER_OBS, WALKER_ACT = 24, 6  # dm_control walker/run (learner.py:24-26), used when dm_control is absent


def _env_sizes():
    """(obs_size, n_actions).  The reference builds a dm_control env only to read these (learner.py:24-26)."""
    if "R2D2_OBS_SIZE" in os.environ:
        return int(os.environ["R2D2_OBS_SIZE"]), int(os.environ["R2D2_N_ACTIONS"])
    try:
        from dm_control import suite
        env = suite.load(domain_name="walker", task_name="run")
        return get_obs(env.reset().observation).shape[1], env.action_spec().shape[0]
    except ImportError:
        return WALKER_OBS, WALKER_ACT


SNAPSHOT_INTERVAL_STEP = 50    # memory_update_interval: snapshots are taken after an ingest


def snapshot_interval_from_environ(env=None, every=SNAPSHOT_INTERVAL_STEP) -> int:
    """R2D2_REPLAY_SNAPSHOT_INTERVAL: 0 (the default, never) or a positive multiple of `every`."""
    v = (os.environ if env is None else env).get("R2D2_REPLAY_SNAPSHOT_INTERVAL", "0")
    try:
        n = int(v)
    except (TypeError, ValueError):
        n = -1
    if n < 0 or n % every:
        raise ValueError("R2D2_REPLAY_SNAPSHOT_INTERVAL must be 0 (never) or a positive multiple of %d (the learner "
                         "steps between ingests), got %r" % (every, v))
    return n


def snapshot_steps(root) -> list:
    """[(step, directory)] of the snapshot directories under `root`, oldest first."""
    if not os.path.isdir(root):
        return []
    out = []
    for name in os.listdir(root):
        m = re.fullmatch(r"step(\d+)", name)
        if m and os.path.isdir(os.path.join(root, name)):
            out.append((int(m.group(1)), os.path.join(root, name)))
    return sorted(out)


def latest_complete_snapshot(root):
    """(step, directory) of the newest snapshot whose COMPLETE marker exists, or None."""
    done = [s for s in snapshot_steps(root) if os.path.isfile(os.path.join(s[1], "COMPLETE"))]
    return done[-1] if done else None


def _write_synced(path, write):
    """write(tmp) then fsync and rename into place: a path that exists is whole."""
    tmp = "%s.tmp%d" % (path, os.getpid())
    write(tmp)
    with open(tmp, "rb+") as f:
        os.fsync(f.fileno())
    os.replace(tmp, path)


def learner_process(n_actors):
    learner = Learner(n_actors)
    learner.run()


class Learner:
    def __init__(self, n_actors, hidden=None, batch_size=None, device=None):
        from r2d2_b200.engine import LearnerEngine, PathConfig
        from r2d2_b200.dist_env import DistEnv
        self.dist_env = DistEnv.from_environ()
        if self.dist_env.distributed:                      # one learner process per GPU
            device = torch.device("cuda:{}".format(self.dist_env.local_rank))
            torch.cuda.set_device(device)
            self.dist_env.init_process_group("nccl", device=device)
        self.obs_size, self.n_actions = _env_sizes()
        self.n_actors = n_actors
        if not self.dist_env.owned_actors(n_actors):
            raise ValueError("rank {} of {} owns no actor: launch at most n_actors = {} learner ranks".format(
                self.dist_env.rank, self.dist_env.world, n_actors))
        self.burn_in_length = 20
        self.learning_length = 40
        self.sequence_length = self.burn_in_length + self.learning_length
        self.n_step = 5
        self.memory_sequence_size = 5000000
        self.batch_size = batch_size or int(os.environ.get("R2D2_BATCH", 32))
        self.hidden = hidden or int(os.environ.get("R2D2_HIDDEN", 128))
        self.model_path = './model_data/'
        self.memory_path = './memory_data/'
        self.model_save_interval = 50
        self.memory_update_interval = 50
        self.replay_snapshot_interval = snapshot_interval_from_environ(every=self.memory_update_interval)
        self.target_update_inverval = int(os.environ.get("R2D2_TARGET_INTERVAL", 500))
        if self.target_update_inverval < 1:
            raise ValueError("R2D2_TARGET_INTERVAL must be >= 1, got {}".format(self.target_update_inverval))
        self.gamma, self.actor_lr, self.critic_lr = 0.997, 1e-4, 1e-3
        self.priority_exponent = float(os.environ.get("R2D2_PRIORITY_EXPONENT", 1.0))
        self.is_exponent = float(os.environ.get("R2D2_IS_EXPONENT", 0.0))
        self.target_tau = float(os.environ.get("R2D2_TARGET_TAU", 1.0))
        self.grad_clip_norm = float(os.environ.get("R2D2_GRAD_CLIP", 0.0))
        self.replay_state_dtype = self._replay_state_dtype_from_environ()
        self.replay_host_gb = self._replay_host_gb_from_environ()
        from r2d2_b200 import td3_options, td_options
        self.td_options = td_options.from_environ()
        self.td3_options = td3_options.from_environ()
        from r2d2_b200 import obs_norm
        self.obs_norm, self.obs_norm_clip = obs_norm.from_environ()
        from r2d2_b200 import metrics
        self.metrics_on = metrics.from_environ()
        self.metrics_path = self.model_path + 'metrics/learner_rank{}.csv'.format(self.dist_env.rank)
        cfg = PathConfig(obs=self.obs_size, act=self.n_actions, hidden=self.hidden, batch=self.batch_size,
                         burn_in=self.burn_in_length, learning=self.learning_length, n_step=self.n_step,
                         gamma=self.gamma, actor_lr=self.actor_lr, critic_lr=self.critic_lr,
                         target_interval=self.target_update_inverval, priority_exponent=self.priority_exponent,
                         is_exponent=self.is_exponent, target_tau=self.target_tau, grad_clip_norm=self.grad_clip_norm,
                         value_rescaling=self.td_options.value_rescaling, rescaling_eps=self.td_options.rescaling_eps,
                         priority_metric=self.td_options.priority_metric, **self.td3_options,
                         global_sampling=self._global_sampling_from_environ(),
                         replay_state_dtype=self.replay_state_dtype,
                         replay_state_memory="host" if self.replay_host_gb > 0 else "device",
                         obs_norm=self.obs_norm, obs_norm_clip=self.obs_norm_clip, metrics=self.metrics_on)
        self.engine = LearnerEngine(cfg, device=device)
        self.engine.enable_data_parallel()
        self.memory = LearnerReplayMemory(memory_sequence_size=self.memory_sequence_size, batch_size=self.batch_size,
                                          obs_size=self.obs_size, n_actions=self.n_actions, hidden=self.hidden,
                                          device=self.engine.device, priority_exponent=self.priority_exponent,
                                          state_dtype=self.replay_state_dtype, host_gb=self.replay_host_gb)
        self.memory.obs_norm = getattr(self.engine, "obs_norm", None)   # None unless R2D2_OBS_NORM=1
        self.state_path = self.model_path + 'learner_state.pt'
        self.snapshot_root = self.model_path + 'replay_snapshot/'
        if os.environ.get("R2D2_RESUME", "0") == "1":
            snap = latest_complete_snapshot(self.snapshot_root)
            if snap is not None:
                self.resume_from_snapshot(*snap)
            elif os.path.isfile(self.state_path):
                self.load_checkpoint()                     # every rank loads the same file: replicas stay identical
        self.save_model()

    @staticmethod
    def _global_sampling_from_environ():
        v = os.environ.get("R2D2_GLOBAL_SAMPLING", "0")
        if v not in ("0", "1"):
            raise ValueError("R2D2_GLOBAL_SAMPLING must be 0 or 1, got {!r}".format(v))
        return v == "1"

    @staticmethod
    def _replay_state_dtype_from_environ():
        v = os.environ.get("R2D2_REPLAY_STATE_DTYPE", "float32")
        if v not in ("float32", "float16"):
            raise ValueError("R2D2_REPLAY_STATE_DTYPE must be float32 or float16, got {!r}".format(v))
        return v

    @staticmethod
    def _replay_host_gb_from_environ():
        v = os.environ.get("R2D2_REPLAY_HOST_GB", "0")
        try:
            gb = float(v)
        except (TypeError, ValueError):
            gb = float("nan")
        if not (math.isfinite(gb) and gb >= 0):
            raise ValueError("R2D2_REPLAY_HOST_GB must be a finite number of GB >= 0 (0 = recurrent states in HBM), "
                             "got {!r}".format(v))
        return gb

    def save_checkpoint(self):
        """Resumable state next to model.pt: nets + both Adam moment sets + step counter (the reference's model.pt has
        weights only, learner.py:56-61, and its learner never loads).  model.pt keeps the reference's format for actors."""
        if not self.dist_env.is_main:
            return
        tmp = self.state_path + '.tmp{}'.format(os.getpid())
        torch.save(self.engine.training_state(), tmp)
        os.replace(tmp, self.state_path)

    def load_checkpoint(self):
        self.engine.load_training_state(torch.load(self.state_path, map_location="cpu"))

    def _shard_path(self, d):
        return os.path.join(d, "shard{}of{}".format(self.dist_env.rank, self.dist_env.world))

    def resume_from_snapshot(self, step, d):
        """The training state of snapshot directory `d` (step `step`), this rank's shard and its CUDA RNG state."""
        shard = self._shard_path(d)
        if not os.path.isfile(shard):
            worlds = sorted({m.group(1) for m in (re.fullmatch(r"shard\d+of(\d+)", f) for f in os.listdir(d)) if m})
            raise ValueError("replay snapshot {} was written at world size {}, this run has world size {} (re-sharding "
                             "a replay is not supported)".format(d, " / ".join(worlds) or "?", self.dist_env.world))
        self.engine.load_training_state(torch.load(os.path.join(d, "learner_state.pt"), map_location="cpu"))
        self.memory.load_snapshot(shard, world=self.dist_env.world)
        if self.dist_env.is_main:
            print("learner: resuming from the replay snapshot of step {} ({} sequences)".format(
                step, self.memory.sequence_counter))

    def save_replay_snapshot(self):
        """./model_data/replay_snapshot/step{N}/ at the current step N: learner_state.pt, every rank's shard, then
        COMPLETE; the older directories go once it is complete."""
        step = self.engine.step_count
        d = os.path.join(self.snapshot_root, "step{}".format(step))
        dist = getattr(self.engine, "_dist", None)
        barrier = dist.barrier if dist is not None else (lambda: None)
        if self.dist_env.is_main:
            for _, old in snapshot_steps(self.snapshot_root):      # an unfinished one from a stopped run
                if old != d and not os.path.isfile(os.path.join(old, "COMPLETE")):
                    shutil.rmtree(old, ignore_errors=True)
            os.makedirs(d, exist_ok=True)
            if os.path.isfile(os.path.join(d, "COMPLETE")):
                os.remove(os.path.join(d, "COMPLETE"))
            state = self.engine.training_state()
            _write_synced(os.path.join(d, "learner_state.pt"), lambda p: torch.save(state, p))
        barrier()
        self.memory.save_snapshot(self._shard_path(d), world=self.dist_env.world, rank=self.dist_env.rank,
                                  learner_step=step)
        barrier()
        if self.dist_env.is_main:
            def mark(p):
                with open(p, "w") as f:
                    f.write("{}\n".format(step))
            _write_synced(os.path.join(d, "COMPLETE"), mark)
            for _, old in snapshot_steps(self.snapshot_root):
                if old != d:
                    shutil.rmtree(old, ignore_errors=True)

    # the four nets as state_dict-compatible views of the engine's flat parameter blocks
    def _sd(self, net):
        return {k: v.detach().clone() for k, v in self.engine.views(net).items()}

    def save_model(self):
        """model.pt = {'actor','target_actor','critic','target_critic'} state_dicts (learner.py:56-61).
        Replicas are identical: rank 0 alone writes."""
        if not self.dist_env.is_main:
            return
        model_dict = {net: self._sd(net) for net in ('actor', 'target_actor', 'critic', 'target_critic')}
        stats = getattr(self.engine, "obs_norm", None)
        norm = stats.actor_key() if stats is not None else None
        if norm is not None:
            model_dict['obs_norm'] = norm
        tmp = self.model_path + 'model.pt.tmp{}'.format(os.getpid())
        torch.save(model_dict, tmp)
        os.replace(tmp, self.model_path + 'model.pt')

    def update_target_model(self):
        self.engine.flush()
        self.engine.discard_prefetched()      # target chains that already ran for the next batch used the old target nets
        self.engine.flat['target_actor'].copy_(self.engine.flat['actor'])
        self.engine.flat['target_critic'].copy_(self.engine.flat['critic'])   # twin critic: the whole [1 | 2] block

    def log_metrics(self):
        """With R2D2_METRICS=1: append the iterations finished since the last call to this rank's CSV file; rank 0
        prints their summary.  A deferred data-parallel finish phase is not forced: its iteration comes next time."""
        m = getattr(self.engine, "metrics", None)
        if m is None:
            return
        from r2d2_b200 import metrics
        rec = m.read()
        if not len(rec["iteration"]):
            return
        metrics.append_records(self.metrics_path, rec)
        if self.dist_env.is_main:
            print(metrics.summary_line(rec))

    def _ingest(self):
        for i in self.dist_env.owned_actors(self.n_actors):   # all of them in a single-process run (learner.py:70-73)
            if os.path.isfile(self.memory_path + '/memory{}.pt'.format(i)):
                self.memory.load(i)

    def run(self, max_steps=None):
        from r2d2_b200.run_loop import run_learner_loop, warm_up

        def report():
            if self.dist_env.is_main:
                print('learner memory sequence size:', self.memory.sequence_counter)
        warm_up(self._ingest, lambda: self.memory.sequence_counter >= self.batch_size * 100,   # learner.py:69-75
                pause=lambda: sleep(0.1), report=report)

        def save():
            self.save_model()
            if os.environ.get("R2D2_SAVE_STATE", "1") == "1":
                self.save_checkpoint()

        def log(step):
            if self.dist_env.is_main:
                print('learning step:', step)
            self.log_metrics()

        ingest = self._ingest
        if self.engine.cfg.global_sampling:
            # every draw waits (bounded) for every rank's shard root: the ranks enter the loop together, and a slow
            # rank's file ingest must not leave its peers' draw kernels spinning - a host barrier after each ingest
            if self.memory._dev.group is None:                   # a second run() keeps the first one's group
                self.memory._dev.attach_group(self.engine)
            barrier = self.engine._dist.barrier if self.engine._dist is not None else (lambda: None)
            barrier()

            def ingest():
                self._ingest()
                barrier()
        snap = {}
        if self.replay_snapshot_interval:
            snap = dict(snapshot=self.save_replay_snapshot, snapshot_every=self.replay_snapshot_interval)
        if getattr(self.engine, "obs_norm", None) is not None:
            snap["exchange"] = self.engine.obs_norm.exchange
        run_learner_loop(self.engine, self.memory._dev, max_steps=max_steps, ingest_every=self.memory_update_interval,
                         save_every=self.model_save_interval, ingest=ingest, save=save, log=log, **snap)
        self.log_metrics()
        torch.cuda.synchronize()

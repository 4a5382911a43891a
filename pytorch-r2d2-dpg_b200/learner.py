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
replay is not part of the checkpoint, so the setting may change across a resume.
"""
import os
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
        self.target_update_inverval = int(os.environ.get("R2D2_TARGET_INTERVAL", 500))
        if self.target_update_inverval < 1:
            raise ValueError("R2D2_TARGET_INTERVAL must be >= 1, got {}".format(self.target_update_inverval))
        self.gamma, self.actor_lr, self.critic_lr = 0.997, 1e-4, 1e-3
        self.priority_exponent = float(os.environ.get("R2D2_PRIORITY_EXPONENT", 1.0))
        self.is_exponent = float(os.environ.get("R2D2_IS_EXPONENT", 0.0))
        self.target_tau = float(os.environ.get("R2D2_TARGET_TAU", 1.0))
        self.grad_clip_norm = float(os.environ.get("R2D2_GRAD_CLIP", 0.0))
        self.replay_state_dtype = self._replay_state_dtype_from_environ()
        from r2d2_b200 import td3_options, td_options
        self.td_options = td_options.from_environ()
        self.td3_options = td3_options.from_environ()
        cfg = PathConfig(obs=self.obs_size, act=self.n_actions, hidden=self.hidden, batch=self.batch_size,
                         burn_in=self.burn_in_length, learning=self.learning_length, n_step=self.n_step,
                         gamma=self.gamma, actor_lr=self.actor_lr, critic_lr=self.critic_lr,
                         target_interval=self.target_update_inverval, priority_exponent=self.priority_exponent,
                         is_exponent=self.is_exponent, target_tau=self.target_tau, grad_clip_norm=self.grad_clip_norm,
                         value_rescaling=self.td_options.value_rescaling, rescaling_eps=self.td_options.rescaling_eps,
                         priority_metric=self.td_options.priority_metric, **self.td3_options,
                         global_sampling=self._global_sampling_from_environ(),
                         replay_state_dtype=self.replay_state_dtype)
        self.engine = LearnerEngine(cfg, device=device)
        self.engine.enable_data_parallel()
        self.memory = LearnerReplayMemory(memory_sequence_size=self.memory_sequence_size, batch_size=self.batch_size,
                                          obs_size=self.obs_size, n_actions=self.n_actions, hidden=self.hidden,
                                          device=self.engine.device, priority_exponent=self.priority_exponent,
                                          state_dtype=self.replay_state_dtype)
        self.state_path = self.model_path + 'learner_state.pt'
        if os.environ.get("R2D2_RESUME", "0") == "1" and os.path.isfile(self.state_path):
            self.load_checkpoint()                         # every rank loads the same file: replicas stay identical
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

    # the four nets as state_dict-compatible views of the engine's flat parameter blocks
    def _sd(self, net):
        return {k: v.detach().clone() for k, v in self.engine.views(net).items()}

    def save_model(self):
        """model.pt = {'actor','target_actor','critic','target_critic'} state_dicts (learner.py:56-61).
        Replicas are identical: rank 0 alone writes."""
        if not self.dist_env.is_main:
            return
        model_dict = {net: self._sd(net) for net in ('actor', 'target_actor', 'critic', 'target_critic')}
        tmp = self.model_path + 'model.pt.tmp{}'.format(os.getpid())
        torch.save(model_dict, tmp)
        os.replace(tmp, self.model_path + 'model.pt')

    def update_target_model(self):
        self.engine.flush()
        self.engine.discard_prefetched()      # target chains that already ran for the next batch used the old target nets
        self.engine.flat['target_actor'].copy_(self.engine.flat['actor'])
        self.engine.flat['target_critic'].copy_(self.engine.flat['critic'])   # twin critic: the whole [1 | 2] block

    def _ingest(self):
        for i in self.dist_env.owned_actors(self.n_actors):   # all of them in a single-process run (learner.py:70-73)
            if os.path.isfile(self.memory_path + '/memory{}.pt'.format(i)):
                self.memory.load(i)

    def run(self, max_steps=None):
        while self.memory.sequence_counter < self.batch_size * 100:   # warm-up gate, learner.py:69-75
            self._ingest()
            sleep(0.1)
            if self.dist_env.is_main:
                print('learner memory sequence size:', self.memory.sequence_counter)
        from r2d2_b200.run_loop import run_learner_loop

        def save():
            self.save_model()
            if os.environ.get("R2D2_SAVE_STATE", "1") == "1":
                self.save_checkpoint()

        def log(step):
            if self.dist_env.is_main:
                print('learning step:', step)

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
        run_learner_loop(self.engine, self.memory._dev, max_steps=max_steps, ingest_every=self.memory_update_interval,
                         save_every=self.model_save_interval, ingest=ingest, save=save, log=log)
        torch.cuda.synchronize()

"""Drop-in for the reference's replay_memory.py.

  ReplayMemory          actor-side episode buffer + `save(actorID)` in the reference's file format
                        (replay_memory.py:8-64); pure host code, unchanged contract.
  LearnerReplayMemory   same constructor / attributes / `sample()` 10-tuple / `load(actorID)` as
                        replay_memory.py:67-175, but the storage is a replay shard in HBM with a sum tree
                        (r2d2_b200.engine.DeviceReplay -> csrc/replay.cu).  P(episode, sequence) is
                        proportional to priority[episode][sequence], the law of the reference's two-level
                        WeightedRandomSampler draw (replay_memory.py:95-114).  With a priority exponent alpha
                        (R2D2_PRIORITY_EXPONENT, default 1 = the reference) the shard stores p^alpha instead:
                        `priority[e][s]` reads the stored p^alpha, and a write of p through it stores p^alpha too.
                        With host_gb > 0 (R2D2_REPLAY_HOST_GB) the rows' recurrent states live in pinned host memory
                        and only the rest of each row and the tree take HBM.

File format (actor.py:163-176, replay_memory.py:55-59): torch.save of
  {'replay_memory': deque[list[(obs f32[O], act f32[A], [reward], [terminal])]],
   'recurrent_state': deque[list[[[hx, cx] x 4 nets]]], 'priority': deque[list[float]], 'total_priority': list}.
"""
import math
import numbers
import os
from collections import deque
from time import sleep

import numpy as np
import torch

BURN_IN, LEARNING, N_STEP = 20, 40, 5  # replay_memory.py:18-20,78-81


class ReplayMemory:
    def __init__(self, memory_sequence_size=100000, batch_size=64):
        self.path = './memory_data/'
        self.memory_sequence_size = memory_sequence_size
        self.batch_size = batch_size
        self.memory, self.priority = deque(), deque()
        self.total_priority, self.recurrent_state = deque(), deque()
        self.burn_in_length, self.learning_length, self.n_step = BURN_IN, LEARNING, N_STEP

    def add(self, episode, recurrent_state, priority):
        self.memory.append(episode)
        self.recurrent_state.append(recurrent_state)
        self.priority.append(priority)
        self.total_priority.append(sum(list(priority)))

    def clear(self):
        for d in (self.memory, self.recurrent_state, self.priority, self.total_priority):
            d.clear()

    def size(self):
        return sum(len(ep) for ep in self.memory)

    def save(self, actorID):
        """Write (the reference always overwrites: its append branch tests a file that never exists,
        replay_memory.py:38) and clear.  Written to a temp name and renamed so a concurrently loading
        learner never sees a half-written pickle."""
        payload = {'replay_memory': self.memory, 'recurrent_state': self.recurrent_state,
                   'priority': self.priority, 'total_priority': list(self.total_priority)}
        final = self.path + 'memory{}.pt'.format(actorID)
        tmp = final + '.tmp{}'.format(os.getpid())
        torch.save(payload, tmp)
        os.replace(tmp, final)
        self.clear()


def pack_episode(rows, states, hidden=None):
    """One episode of the actor format -> contiguous float32 arrays (obs, act, rew, term, states[E,4,2,H])."""
    obs = np.stack([np.asarray(r[0], np.float32) for r in rows])
    act = np.stack([np.asarray(r[1], np.float32) for r in rows])
    rew = np.asarray([r[2][0] for r in rows], np.float32)
    term = np.asarray([r[3][0] for r in rows], np.float32)
    st = np.asarray(states, np.float32)  # [E, 4, 2, H]
    if st.ndim != 4 or st.shape[1:3] != (4, 2):
        raise ValueError("recurrent_state must be [steps][4 nets][hx, cx][H], got %r" % (st.shape,))
    if hidden is not None and st.shape[3] != hidden:
        raise ValueError("recurrent state width %d != hidden %d" % (st.shape[3], hidden))
    return obs, act, rew, term, st


class _EpisodePriorities:
    """`memory.priority[e]`: indexable / assignable view of one episode's leaf priorities in HBM.  Reads give the stored
    leaf, p^alpha under a priority exponent; an assigned raw p goes through update_priorities and is raised as well."""

    def __init__(self, owner, e):
        self._o, self._e = owner, e

    def __len__(self):
        return self._o._episodes[self._e][2]

    def _row(self, s):
        start, _, n_starts = self._o._episodes[self._e]
        if s < 0:
            s += n_starts
        if not 0 <= s < n_starts:
            raise IndexError(s)
        return start + s

    def __getitem__(self, s):
        return float(self._o._dev.tree_level(0)[self._row(s)].item())

    def __setitem__(self, s, value):
        o = self._o
        leaf = torch.tensor([self._row(s)], dtype=torch.int64, device=o._dev.device)
        o._dev.update_priorities(leaf, torch.tensor([float(value)], dtype=torch.float32, device=o._dev.device))

    def __iter__(self):
        start, _, n_starts = self._o._episodes[self._e]
        return iter(self._o._dev.tree_level(0)[start:start + n_starts].cpu().tolist())


class _PriorityTable:
    def __init__(self, owner):
        self._o = owner

    def __len__(self):
        return len(self._o._episodes)

    def __getitem__(self, e):
        return _EpisodePriorities(self._o, e)


class _TotalPriority:
    """`memory.total_priority[e]`: the tree maintains the sums, so assignment is accepted and ignored
    (learner.py:139 recomputes it from priority[e] after every write)."""

    def __init__(self, owner):
        self._o = owner

    def __len__(self):
        return len(self._o._episodes)

    def __getitem__(self, e):
        return float(sum(_EpisodePriorities(self._o, e)))

    def __setitem__(self, e, value):
        pass


class LearnerReplayMemory:
    def __init__(self, memory_sequence_size=500000, batch_size=32, obs_size=None, n_actions=None, hidden=128,
                 capacity_rows=None, device=None, priority_exponent=None, state_dtype="float32", host_gb=0):
        self.path = './memory_data/'
        self.memory_sequence_size = memory_sequence_size
        self.sequence_counter = 0
        self.batch_size = batch_size
        self.burn_in_length, self.learning_length, self.n_step = BURN_IN, LEARNING, N_STEP
        self.sequence_length = self.burn_in_length + self.learning_length
        self._hidden, self._obs, self._act = hidden, obs_size, n_actions
        self._capacity_rows, self._device = capacity_rows, device
        if priority_exponent is None:
            priority_exponent = float(os.environ.get("R2D2_PRIORITY_EXPONENT", 1.0))
        self.priority_exponent = float(priority_exponent)
        self.state_dtype = state_dtype                      # stored recurrent states: "float32" or "float16"
        if isinstance(host_gb, bool) or not isinstance(host_gb, numbers.Real) or not (math.isfinite(host_gb)
                                                                                      and host_gb >= 0):
            raise ValueError("host_gb must be a finite number >= 0 (0 = states in HBM), got %r" % (host_gb,))
        self.host_gb = float(host_gb)                       # > 0: the states live in this much pinned host memory
        self._cfg()                                         # rejects an exponent outside [0, 1] before any ingest
        self._dev = None          # DeviceReplay, created when the row width is known
        self._episodes = deque()  # (row_start, n_rows, n_starts) in FIFO order, mirrors the native ring
        self.obs_norm = None      # ObsNormStats (observation normalisation): ingests feed it, the shard's gathers read it
        self.priority = _PriorityTable(self)
        self.total_priority = _TotalPriority(self)

    # the reference exposes the raw deques; here the rows live in HBM
    @property
    def memory(self):
        return self._episodes

    @property
    def recurrent_state(self):
        return self._episodes

    def size(self):
        return sum(e[1] for e in self._episodes)

    def clear(self):
        if self._dev is not None:
            self._dev.close()
        self._dev = None
        self._episodes.clear()
        self.sequence_counter = 0

    def _cfg(self):
        from r2d2_b200.engine import PathConfig
        return PathConfig(obs=self._obs, act=self._act, hidden=self._hidden, batch=self.batch_size,
                          burn_in=self.burn_in_length, learning=self.learning_length, n_step=self.n_step,
                          priority_exponent=self.priority_exponent, replay_state_dtype=self.state_dtype,
                          replay_state_memory="host" if self.host_gb > 0 else "device")

    def _ensure_device(self, obs_size, n_actions, hidden):
        """Create the HBM shard on first use.  Sizes given to the constructor are binding: an actor file of another
        width is an error, not a silent re-shape (the engine's batch buffers are sized from the same numbers)."""
        for name, want, got in (("obs_size", self._obs, obs_size), ("n_actions", self._act, n_actions),
                                ("hidden", self._hidden, hidden)):
            if want is not None and want != got:
                raise ValueError("actor file %s = %d, learner was built for %d" % (name, got, want))
        if self._dev is None:
            from r2d2_b200.engine import DeviceReplay
            self._obs, self._act, self._hidden = obs_size, n_actions, hidden
            rows = self._capacity_rows or self._default_capacity_rows(obs_size, n_actions, hidden)
            self._dev = DeviceReplay(self._cfg(), capacity_rows=rows, max_sequences=self.memory_sequence_size,
                                     device=self._device)
            if self.obs_norm is not None:
                self._dev.attach_obs_norm(self.obs_norm)
        return self._dev

    def _default_capacity_rows(self, obs_size, n_actions, hidden):
        """Ring rows for `memory_sequence_size` sequences (one stored row per sequence start plus the 64 rows per
        episode that start no sequence: x1.3), capped at 60 % of the free HBM.  The reference keeps up to
        memory_sequence_size sequences in host RAM (replay_memory.py:148); when the cap applies, FIFO eviction starts
        earlier than there - said out loud, and documented in INTEGRATION.md.  fp16 state storage halves the
        recurrent states [4,2,H] of a row, so the same cap holds nearly twice the rows.

        With host_gb > 0 the states live in pinned host memory: a row then takes 4 (O + A + 2) + 5 bytes of HBM and
        16 H (fp16) or 32 H (fp32) bytes of host memory, and the ring is the least of the wanted rows, the rows that fit
        60 % of the free HBM and the rows that fit host_gb * 1e9 bytes; the note names the limit that applies."""
        want = int(self.memory_sequence_size * 1.3) + 4096
        state_bytes = 16 if self.state_dtype == "float16" else 32              # (h, c) of four nets, per unit of H
        if self.host_gb > 0:
            return self._host_tier_capacity_rows(want, obs_size, n_actions, state_bytes * hidden)
        bytes_per_row = 4 * (obs_size + n_actions + 2) + state_bytes * hidden + 5   # rows + leaf + ancestors
        free = torch.cuda.mem_get_info(self._device)[0] if torch.cuda.is_available() else 0
        fit = int(0.6 * free / bytes_per_row)
        if 0 < fit < want:
            print("LearnerReplayMemory: ring capped at %d rows (%.1f GB of HBM, %s recurrent states) for "
                  "memory_sequence_size=%d; FIFO eviction starts earlier than the reference's"
                  % (fit, fit * bytes_per_row / 1e9, self.state_dtype, self.memory_sequence_size))
            return fit
        return want

    def _host_tier_capacity_rows(self, want, obs_size, n_actions, host_row):
        hbm_row = 4 * (obs_size + n_actions + 2) + 5                           # rows + leaf + ancestors
        free = torch.cuda.mem_get_info(self._device)[0] if torch.cuda.is_available() else 0
        limits = [(want, "memory_sequence_size=%d" % self.memory_sequence_size)]
        if free > 0:
            limits.append((int(0.6 * free / hbm_row), "60 %% of the free HBM (%.1f GB)" % (free / 1e9)))
        limits.append((int(self.host_gb * 1e9 / host_row), "the host budget host_gb=%g" % self.host_gb))
        rows, limit = min(limits, key=lambda x: x[0])
        if rows < 1:
            raise ValueError("LearnerReplayMemory: %s holds no replay row (%d bytes of %s recurrent states per row)"
                             % (limit, host_row, self.state_dtype))
        print("LearnerReplayMemory: ring of %d rows, limited by %s: %.2f GB of HBM (%d bytes per row) and %.2f GB of "
              "pinned host memory (%s recurrent states, %d bytes per row)%s"
              % (rows, limit, rows * hbm_row / 1e9, hbm_row, rows * host_row / 1e9, self.state_dtype, host_row,
                 "" if rows == want else "; FIFO eviction starts earlier than the reference's"))
        return rows

    def _register(self, starts, n_rows, n_starts, n_evicted, counter):
        """Mirror of the native FIFO: evictions (ring overlap while appending, sequence cap afterwards) always take the
        oldest episode, so the survivors are (old + new) minus the first `n_evicted`."""
        for st, nr, ns in zip(starts, n_rows, n_starts):
            self._episodes.append((int(st), int(nr), int(ns)))
        for _ in range(min(int(n_evicted), len(self._episodes))):
            self._episodes.popleft()
        self.sequence_counter = int(counter)

    def save_snapshot(self, path, world=1, rank=0, learner_step=0, **kw):
        """The HBM shard and the CUDA RNG state to one file (r2d2_b200.replay_snapshot); nothing to save before the
        first ingest."""
        if self._dev is None:
            raise ValueError("LearnerReplayMemory.save_snapshot: the replay holds nothing yet")
        return self._dev.save_snapshot(path, world=world, rank=rank, learner_step=learner_step, **kw)

    def load_snapshot(self, path, world=None, restore_rng=True, **kw):
        """Restore a snapshot into an empty replay.  The device shard is created from the file's sizes if none exists
        yet (sizes given to the constructor stay binding), with this replay's capacity and state storage: another ring
        size compacts the episodes, another storage type is converted.  `priority[e]`, `sample()` and `decode` then
        see the saved shard.  Returns the snapshot's header fields (replay_snapshot.load)."""
        from r2d2_b200 import replay_snapshot
        if self._episodes:
            raise ValueError("LearnerReplayMemory.load_snapshot: the replay is not empty")
        with open(path, "rb") as f:
            h = replay_snapshot.Header.read(f)
        if (h.burn_in, h.learning, h.n_step) != (self.burn_in_length, self.learning_length, self.n_step):
            raise ValueError("replay snapshot %s has burn-in / learning / n-step %r, this replay %r" % (
                path, (h.burn_in, h.learning, h.n_step), (self.burn_in_length, self.learning_length, self.n_step)))
        dev = self._ensure_device(h.obs_size, h.n_actions, h.hidden)
        out = dev.load_snapshot(path, world=world, restore_rng=restore_rng, **kw)
        rs, nr, ns, _ = dev.episodes()
        self._episodes = deque((int(a), int(b), int(c)) for a, b, c in zip(rs, nr, ns))
        self.sequence_counter = int(dev.snapshot_info()["sequence_counter"])
        return out

    def add_episode(self, rows, states, priority):
        obs, act, rew, term, st = pack_episode(rows, states, self._hidden)
        dev = self._ensure_device(obs.shape[1], act.shape[1], st.shape[3])
        starts, n_evicted, counter = dev.add_episodes([(obs, act, rew, term, st, np.asarray(priority, np.float32))],
                                                      obs_norm=self.obs_norm)
        self._register(starts, [obs.shape[0]], [len(priority)], n_evicted, counter)

    def get_weighted_sample_index(self):
        """Iterator of `batch_size` episode indices drawn proportionally to the episode totals
        (replay_memory.py:95-97), realised as the episode component of flat tree draws."""
        u = torch.rand(self.batch_size, device=self._dev.device)
        ep, _ = self._dev.decode(self._dev.sample_indices(u))
        return iter(int(e) for e in ep)

    def sample(self):
        """Same 10-tuple as replay_memory.py:99-136 (lists of ints + time-major CUDA tensors)."""
        B, T = self.batch_size, self.sequence_length + self.n_step
        dev = self._dev
        d = dev.device
        u = torch.rand(B, device=d)
        leaf = torch.empty(B, dtype=torch.int64, device=d)
        obs = torch.empty((T, B, self._obs), device=d)
        act = torch.empty((T, B, self._act), device=d)
        rew = torch.empty((T, B, 1), device=d)
        term = torch.empty((T, B, 1), device=d)
        states = torch.empty((4, 2, B, self._hidden), device=d)
        from r2d2_b200 import native as nv
        nv.check(dev.lib.r2d2_replay_sample(dev._h, nv.dptr(u), B, nv.dptr(leaf, torch.int64), nv.dptr(obs),
                                            nv.dptr(act), nv.dptr(rew), nv.dptr(term), nv.dptr(states),
                                            nv.current_stream()))
        ep, seq = dev.decode(leaf)
        return ([int(e) for e in ep], [int(s) for s in seq], obs, act, rew, term,
                states[0], states[1], states[2], states[3])

    def load(self, actorID):
        """Ingest memory{actorID}.pt (replay_memory.py:138-157): all episodes of the file are appended, then the oldest
        are dropped while the sequence counter exceeds memory_sequence_size.

        Differences from the reference, deliberate: (1) the file is CLAIMED by an atomic rename before it is read and
        removed afterwards (the reference reads it, then rewrites it emptied: an actor's fresh file saved in between is
        overwritten and its episodes are lost; an emptied file and no file are the same to `learner.py:70-73`, which tests
        `isfile` first); (2) the whole payload is parsed and validated BEFORE anything is ingested and goes to the
        device in one native call - a failure cannot leave half a file in the shard, so the reference's retry (one
        more attempt after a pause, replay_memory.py:158-175) never duplicates episodes; malformed episodes are skipped;
        (3) weights_only=False: the payload is a pickle of deques / ndarrays, which torch >= 2.6 refuses by default."""
        fname = self.path + 'memory{}.pt'.format(actorID)
        if not os.path.isfile(fname):
            return
        claimed = fname + '.ingest{}'.format(os.getpid())
        try:
            os.replace(fname, claimed)
        except OSError:
            return                                          # another process took it, or the actor is mid-rename
        payload = None
        for attempt in (0, 1):
            try:
                payload = torch.load(claimed, weights_only=False)
                break
            except Exception:
                if attempt:
                    os.replace(claimed, fname)              # hand the file back untouched
                    raise
                sleep(np.random.rand() * 5 + 2)
        episodes = []
        for rows, states, prio in zip(payload['replay_memory'], payload['recurrent_state'], payload['priority']):
            if len(rows) < self.sequence_length + self.n_step:
                continue
            try:
                obs, act, rew, term, st = pack_episode(rows, states, self._hidden)
            except (ValueError, TypeError, IndexError) as exc:
                print("LearnerReplayMemory.load: skipping a malformed episode of {}: {}".format(fname, exc))
                continue
            episodes.append((obs, act, rew, term, st, np.asarray(prio, np.float32)))
        if episodes:
            dev = self._ensure_device(episodes[0][0].shape[1], episodes[0][1].shape[1], episodes[0][4].shape[3])
            starts, n_evicted, counter = dev.add_episodes(episodes, obs_norm=self.obs_norm)
            self._register(starts, [e[0].shape[0] for e in episodes], [len(e[5]) for e in episodes], n_evicted, counter)
        os.remove(claimed)

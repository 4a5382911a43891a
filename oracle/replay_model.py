"""Host model of one replay shard (pytorch-r2d2-dpg_b200/csrc/replay.cu) in plain numpy - TEST INFRASTRUCTURE.

It restates what a shard should hold from the rules the shard documents, not from its code, so that the tests can
compare a DeviceReplay with it after every ingest, write-back and restore:

- Placement: an episode of n rows goes at `head`; when head + n exceeds the capacity it goes at row 0 instead (the tail
  gap stays unused).  Then the oldest live episodes are evicted, front first, until none overlaps [start, start + n) -
  after a wrap that can be an old episode at the tail and younger ones at the head.
- One call (an actor file) places and writes its episodes in order; only after the whole call are the oldest episodes
  evicted while the sequence counter exceeds max_sequences (0: no cap), down to an empty shard if need be - the
  reference's LearnerReplayMemory.load (replay_memory.py:138-157).  A single-episode call follows the same rules.
- The sequence counter grows by n - (W - 1) per stored episode (W = burn_in + learning + n_step, replay_memory.py:147)
  and shrinks by n - (burn_in + learning) per evicted one (:149): the reference's asymmetric count.
- Leaves: row r of a live episode holds priority^alpha on its first n_starts rows (0 stays 0; alpha = 1 keeps the
  value as given) and 0 on every other row of the ring.  A write-back applies its entries in batch order, so the last
  writer of a duplicate leaf wins.
- Rows hold obs / act / rew / term and the recurrent states of the episode's rows (zero past the states given,
  rounded to fp16 with round-to-nearest-even in fp16 storage).  An evicted episode's rows stay until overwritten.
- A snapshot restored at the same capacity is the same shard (rows outside the live episodes zero).  At another
  capacity the oldest episodes are dropped while the rest does not fit, counted as evictions, and the survivors are
  packed from row 0 in FIFO order.
"""
from __future__ import annotations

from collections import deque

import numpy as np

TREE_K = 32


class ReplayModel:
    def __init__(self, capacity: int, obs: int, act: int, hidden: int, burn_in: int, learning: int, n_step: int,
                 max_sequences: int = 0, alpha: float = 1.0, state_f16: bool = False):
        self.capacity = int(capacity)
        self.obs_size, self.n_actions, self.hidden = int(obs), int(act), int(hidden)
        self.burn_in, self.learning, self.n_step = int(burn_in), int(learning), int(n_step)
        self.rows_per_window = self.burn_in + self.learning + self.n_step
        self.max_sequences = int(max_sequences)
        self.alpha = float(alpha)
        self.state_f16 = bool(state_f16)
        cap = self.capacity
        self.obs = np.zeros((cap, self.obs_size), np.float32)
        self.act = np.zeros((cap, self.n_actions), np.float32)
        self.rew = np.zeros(cap, np.float32)
        self.term = np.zeros(cap, np.float32)
        self.states = np.zeros((cap, 4, 2, self.hidden), np.float32)
        self.raw = np.zeros(cap, np.float32)        # the priority behind every leaf, as given
        self.fifo = deque()                          # [row_start, n_rows, n_starts, serial], oldest first
        self.head = self.sequence_counter = self.rows_used = self.next_serial = self.evicted_total = 0

    @classmethod
    def for_config(cls, cfg, capacity: int, max_sequences: int = 0) -> "ReplayModel":
        """The model of DeviceReplay(cfg, capacity, max_sequences); cfg has PathConfig's fields."""
        return cls(capacity, cfg.obs, cfg.act, cfg.hidden, cfg.burn_in, cfg.learning, cfg.n_step, max_sequences,
                   cfg.priority_exponent, cfg.replay_state_dtype == "float16")

    # ---- ingest --------------------------------------------------------------------------------------------------
    def _evict_front(self):
        s, n, k, _ = self.fifo.popleft()
        self.raw[s:s + k] = 0
        self.sequence_counter -= n - (self.burn_in + self.learning)
        self.rows_used -= n
        self.evicted_total += 1

    def _place(self, n: int) -> int:
        if self.head + n > self.capacity:
            self.head = 0
        start, end = self.head, self.head + n
        while any(s < end and start < s + m for s, m, _, _ in self.fifo):
            self._evict_front()
        return start

    def add_episodes(self, episodes):
        """One call of DeviceReplay.add_episodes: episodes are (obs [n,O], act [n,A], rew [n], term [n],
        states [n_real,4,2,H], priority [n_starts]).  Returns (row start per episode, episodes evicted by the call,
        sequence counter)."""
        evicted0 = self.evicted_total
        starts = []
        for obs, act, rew, term, states, prio in episodes:
            obs = np.asarray(obs, np.float32)
            prio = np.asarray(prio, np.float32).reshape(-1)
            states = np.asarray(states, np.float32).reshape(-1, 4, 2, self.hidden)
            n, k, W = obs.shape[0], prio.size, self.rows_per_window
            if not (W <= n <= self.capacity and k <= n - W + 1 and k <= states.shape[0] <= n):
                raise ValueError("episode of %d rows, %d starts, %d state rows does not fit the shard"
                                 % (n, k, states.shape[0]))
            s = self._place(n)
            self.obs[s:s + n] = obs
            self.act[s:s + n] = np.asarray(act, np.float32)
            self.rew[s:s + n] = np.asarray(rew, np.float32).reshape(-1)
            self.term[s:s + n] = np.asarray(term, np.float32).reshape(-1)
            st = np.zeros((n, 4, 2, self.hidden), np.float32)
            st[:states.shape[0]] = states
            self.states[s:s + n] = st.astype(np.float16).astype(np.float32) if self.state_f16 else st
            self.raw[s:s + n] = 0
            self.raw[s:s + k] = prio
            self.fifo.append([s, n, k, self.next_serial])
            self.next_serial += 1
            self.head = s + n
            self.rows_used += n
            self.sequence_counter += n - (self.rows_per_window - 1)
            starts.append(s)
        while self.max_sequences > 0 and self.sequence_counter > self.max_sequences and self.fifo:
            self._evict_front()
        return starts, self.evicted_total - evicted0, self.sequence_counter

    def add_episode(self, obs, act, rew, term, states, priority):
        """DeviceReplay.add_episode: a call of one episode."""
        return self.add_episodes([(obs, act, rew, term, states, priority)])

    def update_priorities(self, leaf, prio):
        """A write-back of raw priorities, in batch order."""
        for l, p in zip(np.asarray(leaf, np.int64), np.asarray(prio, np.float32)):
            self.raw[l] = p

    # ---- what the shard holds ------------------------------------------------------------------------------------
    def leaves(self) -> np.ndarray:
        """Level 0 of the sum tree in float64: the raw priority at alpha = 1, p^alpha for p > 0 otherwise, else 0."""
        raw = self.raw.astype(np.float64)
        if self.alpha == 1.0:
            return raw
        out = np.zeros_like(raw)
        pos = raw > 0
        out[pos] = raw[pos] ** self.alpha
        return out

    def live_starts(self) -> np.ndarray:
        """The sequence-start rows of the live episodes, ascending."""
        rows = [np.arange(s, s + k) for s, _, k, _ in self.fifo]
        return np.sort(np.concatenate(rows)) if rows else np.zeros(0, np.int64)

    def decode(self, leaf):
        """(FIFO index, row within the episode) of every leaf, or (-1, -1) on a row no live episode holds."""
        leaf = np.asarray(leaf, np.int64)
        ep = np.full(leaf.shape, -1, np.int64)
        seq = np.full(leaf.shape, -1, np.int64)
        for i, (s, n, _, _) in enumerate(self.fifo):
            hit = (leaf >= s) & (leaf < s + n)
            ep[hit] = i
            seq[hit] = leaf[hit] - s
        return ep, seq

    def window(self, leaf) -> dict:
        """What a gather at `leaf` returns: obs [T,B,O], act [T,B,A], rew / term [T,B], states [4,2,B,H]."""
        leaf = np.asarray(leaf, np.int64)
        r = leaf[None, :] + np.arange(self.rows_per_window)[:, None]
        return {"obs": self.obs[r], "act": self.act[r], "rew": self.rew[r], "term": self.term[r],
                "states": self.states[leaf].transpose(1, 2, 0, 3)}

    def tree_sizes(self) -> list:
        """Nodes per tree level: the leaves padded to a multiple of 32, then ceil(n / 32) up to the single root."""
        n = -(-self.capacity // TREE_K) * TREE_K
        sizes = [n]
        while n > 1:
            n = -(-n // TREE_K)
            sizes.append(n)
        return sizes

    def stats(self) -> dict:
        """DeviceReplay.stats() without the root's value."""
        sizes = self.tree_sizes()
        return {"n_episodes": len(self.fifo), "n_rows_used": self.rows_used, "sequence_counter": self.sequence_counter,
                "capacity_rows": self.capacity, "tree_levels": len(sizes), "tree_nodes": sum(sizes),
                "last_row_start": self.fifo[-1][0] if self.fifo else -1}

    def info(self) -> dict:
        """The counters of DeviceReplay.snapshot_info()."""
        return {"capacity_rows": self.capacity, "max_sequences": self.max_sequences, "n_episodes": len(self.fifo),
                "head": self.head, "sequence_counter": self.sequence_counter, "next_serial": self.next_serial,
                "evicted_total": self.evicted_total, "rows_used": self.rows_used,
                "priority_exponent": float(np.float32(self.alpha)), "state_storage": int(self.state_f16)}

    def episodes(self):
        """DeviceReplay.episodes(): (row_start, n_rows, n_starts, serial) int64 arrays in FIFO order."""
        t = np.asarray(list(self.fifo), np.int64).reshape(-1, 4)
        return tuple(np.ascontiguousarray(t[:, i]) for i in range(4))

    # ---- snapshot restore ----------------------------------------------------------------------------------------
    def restored(self, capacity: int, max_sequences: int | None = None):
        """(model of a fresh shard of `capacity` rows that restored a snapshot of this one, episodes dropped)."""
        m = ReplayModel(capacity, self.obs_size, self.n_actions, self.hidden, self.burn_in, self.learning, self.n_step,
                        self.max_sequences if max_sequences is None else max_sequences, self.alpha, self.state_f16)
        m.sequence_counter, m.next_serial = self.sequence_counter, self.next_serial
        m.evicted_total, m.rows_used = self.evicted_total, self.rows_used
        kept = list(self.fifo)
        dropped = 0
        same = m.capacity == self.capacity
        if not same:
            while kept and m.rows_used > m.capacity:
                _, n, _, _ = kept.pop(0)
                m.sequence_counter -= n - (self.burn_in + self.learning)
                m.rows_used -= n
                m.evicted_total += 1
                dropped += 1
        at = 0
        for s, n, k, serial in kept:
            d = s if same else at
            m.obs[d:d + n] = self.obs[s:s + n]
            m.act[d:d + n] = self.act[s:s + n]
            m.rew[d:d + n] = self.rew[s:s + n]
            m.term[d:d + n] = self.term[s:s + n]
            m.states[d:d + n] = self.states[s:s + n]
            m.raw[d:d + n] = self.raw[s:s + n]
            m.fifo.append([d, n, k, serial])
            at = d + n
        m.head = self.head if same else at
        return m, dropped

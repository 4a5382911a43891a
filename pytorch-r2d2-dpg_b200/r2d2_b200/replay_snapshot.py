"""Replay shard snapshots: one file per shard, written and read through two fixed pinned staging buffers, so host memory
does not grow with the shard.  Only this module knows the layout (little-endian throughout):

    header   magic "R2D2RPLY", version, header bytes; obs, act, hidden, burn-in, learning, n-step, state storage
             (0 fp32, 1 fp16), alpha (float32); capacity rows, max sequences, episodes, head, sequence counter, next
             serial, evicted total, rows used; world, rank; learner step; rows per chunk; the CUDA RNG state's length,
             then its bytes (the device's default generator, which draws the sampler's uniforms)
    table    one (row_start int64, n_rows int32, n_starts int32, serial int64) per live episode, FIFO order
    rows     the live episodes' rows packed in FIFO order, in chunks of `rows per chunk` rows (the last one shorter);
             a chunk of c rows holds obs [c,O], act [c,A], rew [c], term [c] in float32, states [c,4,2,H] in the
             stored type, and the leaves [c] (p^alpha) in float32

Everything the header promises is checked before the shard is touched: magic, version, sizes, alpha, the world size
when the caller names one, and the file's length, so a truncated file is refused with the shard left as it was.  The
writer fsyncs the file before renaming it into place, so a path that exists always holds a whole snapshot.
"""
from __future__ import annotations

import os
import struct
import time
from concurrent.futures import ThreadPoolExecutor
from ctypes import byref, c_longlong, c_void_p
from dataclasses import dataclass, fields

import numpy as np

MAGIC = b"R2D2RPLY"
VERSION = 1
STAGE_BYTES = 64 << 20                       # each of the two pinned staging buffers

_FIXED = struct.Struct("<8sII7if8qiiqqq")
_EPISODE = np.dtype([("row_start", "<i8"), ("n_rows", "<i4"), ("n_starts", "<i4"), ("serial", "<i8")])
SIZE_FIELDS = ("obs_size", "n_actions", "hidden", "burn_in", "learning", "n_step")


@dataclass
class Header:
    obs_size: int
    n_actions: int
    hidden: int
    burn_in: int
    learning: int
    n_step: int
    state_storage: int
    priority_exponent: float
    capacity_rows: int
    max_sequences: int
    n_episodes: int
    head: int
    sequence_counter: int
    next_serial: int
    evicted_total: int
    rows_used: int
    world: int = 1
    rank: int = 0
    learner_step: int = 0
    chunk_rows: int = 1
    rng_state: bytes = b""

    def to_bytes(self) -> bytes:
        vals = [getattr(self, f.name) for f in fields(self) if f.name != "rng_state"]
        n = _FIXED.size + len(self.rng_state)
        return _FIXED.pack(MAGIC, VERSION, n, *vals, len(self.rng_state)) + self.rng_state

    @classmethod
    def read(cls, f) -> "Header":
        raw = f.read(_FIXED.size)
        if len(raw) < _FIXED.size:
            raise ValueError("replay snapshot %s: truncated header" % _name(f))
        magic, version, n, *vals = _FIXED.unpack(raw)
        if magic != MAGIC:
            raise ValueError("replay snapshot %s: not a replay snapshot (magic %r)" % (_name(f), magic))
        if version != VERSION:
            raise ValueError("replay snapshot %s: format version %d, this build reads version %d" % (_name(f), version,
                                                                                                     VERSION))
        rng_len = vals.pop()
        if n != _FIXED.size + rng_len:
            raise ValueError("replay snapshot %s: header length %d does not match its fields" % (_name(f), n))
        rng = f.read(rng_len)
        if len(rng) < rng_len:
            raise ValueError("replay snapshot %s: truncated header" % _name(f))
        h = cls(*vals, rng_state=rng)
        if h.n_episodes < 0 or h.rows_used < 0 or h.chunk_rows < 1 or h.state_storage not in (0, 1):
            raise ValueError("replay snapshot %s: malformed header" % _name(f))
        return h

    @property
    def header_bytes(self) -> int:
        return _FIXED.size + len(self.rng_state)

    def state_row_bytes(self) -> int:
        """Bytes of one row's recurrent states [4, 2, H] in the stored type."""
        return (2 if self.state_storage else 4) * 8 * self.hidden

    def row_bytes(self) -> int:
        return 4 * (self.obs_size + self.n_actions + 3) + self.state_row_bytes()

    def file_bytes(self) -> int:
        return self.header_bytes + self.n_episodes * _EPISODE.itemsize + self.rows_used * self.row_bytes()

    def sizes(self) -> tuple:
        return tuple(getattr(self, k) for k in SIZE_FIELDS)


def _name(f):
    return getattr(f, "name", "?")


def pack_episodes(row_start, n_rows, n_starts, serial) -> bytes:
    t = np.zeros(len(row_start), _EPISODE)
    t["row_start"], t["n_rows"], t["n_starts"], t["serial"] = row_start, n_rows, n_starts, serial
    return t.tobytes()


def read_episodes(f, h: Header) -> np.ndarray:
    raw = f.read(h.n_episodes * _EPISODE.itemsize)
    if len(raw) != h.n_episodes * _EPISODE.itemsize:
        raise ValueError("replay snapshot %s: truncated episode table" % _name(f))
    return np.frombuffer(raw, _EPISODE).copy()


def check_header(h: Header, path, sizes: tuple, alpha: float, world: int | None = None):
    """Refuses a snapshot the shard cannot take: other sizes, another alpha (the leaves hold p^alpha and the raw
    priorities are not kept), another world size (re-sharding is not supported), or a file shorter or longer than its
    header promises."""
    if h.sizes() != tuple(sizes):
        raise ValueError("replay snapshot %s has obs / act / hidden / burn-in / learning / n-step %r, the shard %r"
                         % (path, h.sizes(), tuple(sizes)))
    if np.float32(h.priority_exponent) != np.float32(alpha):
        raise ValueError("replay snapshot %s was written at priority exponent %r, the shard runs %r (the leaves hold "
                         "p^alpha and the raw priorities are not kept)" % (path, h.priority_exponent, alpha))
    if world is not None and h.world != world:
        raise ValueError("replay snapshot %s was written by a run of world size %d, this run has world size %d "
                         "(re-sharding a replay is not supported)" % (path, h.world, world))
    size = os.path.getsize(path)
    if size != h.file_bytes():
        raise ValueError("replay snapshot %s is %d bytes, its header promises %d: truncated or damaged"
                         % (path, size, h.file_bytes()))


def _chunk_layout(h: Header, c: int):
    """(offset, bytes) of obs, act, rew, term, states, leaves in a chunk of c rows."""
    parts, off = [], 0
    for n in (4 * h.obs_size * c, 4 * h.n_actions * c, 4 * c, 4 * c, h.state_row_bytes() * c, 4 * c):
        parts.append((off, n))
        off += n
    return parts


def _ring_runs(row_start, n_rows):
    """The FIFO's contiguous ring ranges [(first row, rows)]: consecutive episodes share a range unless the ring wrapped."""
    runs = []
    for s, n in zip(row_start.tolist(), n_rows.tolist()):
        if runs and runs[-1][0] + runs[-1][1] == s:
            runs[-1][1] += n
        else:
            runs.append([s, n])
    return runs


def _pinned(nbytes):
    import torch
    return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, pin_memory=True)


class _Clock:
    """Optional split of a save / load: device copies (CUDA events), file I/O (host clock), the tree rebuild (events)."""

    def __init__(self, out):
        self.out = out
        if out is not None:
            out.update(device_s=0.0, io_s=0.0, rebuild_s=0.0)

    def device(self, key, fn):
        if self.out is None:
            return fn()
        import torch
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        rc = fn()
        b.record()
        b.synchronize()
        self.out[key] += a.elapsed_time(b) / 1e3
        return rc

    def io(self, fn):
        t = time.perf_counter()
        r = fn()
        if self.out is not None:
            self.out["io_s"] += time.perf_counter() - t
        return r


def save(dev, path, world: int = 1, rank: int = 0, learner_step: int = 0, stage_bytes: int = STAGE_BYTES,
         timings: dict | None = None):
    """Writes DeviceReplay `dev` to `path` (via path.tmp<pid>, fsynced, then renamed).  The CUDA RNG state of the
    shard's device goes into the header."""
    import torch

    from . import native as nv
    lib, hd = dev.lib, dev._h
    t0 = time.perf_counter()
    clock = _Clock(timings)
    info = nv.ReplaySnapshotInfo()
    nv.check(lib.r2d2_replay_export_info(hd, byref(info)))
    E = int(info.n_episodes)
    rs, nr = np.zeros(E, np.int64), np.zeros(E, np.int32)
    ns, se = np.zeros(E, np.int32), np.zeros(E, np.int64)
    P = lambda a: a.ctypes.data_as(c_void_p)  # noqa: E731
    nv.check(lib.r2d2_replay_export_episodes(hd, P(rs), P(nr), P(ns), P(se)))
    h = Header(**{k: getattr(info, k) for k, _ in nv.ReplaySnapshotInfo._fields_}, world=int(world), rank=int(rank),
               learner_step=int(learner_step),
               rng_state=torch.cuda.get_rng_state(dev.device).numpy().tobytes())
    rb = h.row_bytes()
    h.chunk_rows = max(1, int(stage_bytes) // rb)
    runs = _ring_runs(rs, nr)
    bufs = [_pinned(h.chunk_rows * rb) for _ in range(2)]
    stream = nv.current_stream()
    tmp = "%s.tmp%d" % (path, os.getpid())
    pending = [None, None]
    with open(tmp, "wb") as f, ThreadPoolExecutor(max_workers=1) as pool:
        clock.io(lambda: (f.write(h.to_bytes()), f.write(pack_episodes(rs, nr, ns, se))))
        packed, k, ri, ro = 0, 0, 0, 0          # rows written, chunk index, current run, offset in it
        while packed < h.rows_used:
            c = min(h.chunk_rows, h.rows_used - packed)
            buf = bufs[k % 2]
            if pending[k % 2] is not None:
                pending[k % 2].result()          # the write of two chunks ago still reads this buffer
            base = buf.data_ptr()
            lay = _chunk_layout(h, c)
            done = 0
            while done < c:                      # a chunk may span the ring's wrap: one export per contiguous piece
                first, n = runs[ri]
                take = min(n - ro, c - done)
                ptrs = []
                for (off, nbytes) in lay:
                    ptrs.append(c_void_p(base + off + nbytes // c * done))
                clock.device("device_s", lambda: nv.check(lib.r2d2_replay_export_rows(
                    hd, first + ro, take, *ptrs, stream)))
                done += take
                ro += take
                if ro == n:
                    ri, ro = ri + 1, 0
            view = memoryview(buf.numpy())[:c * rb]
            pending[k % 2] = pool.submit(clock.io, lambda v=view: f.write(v))
            packed += c
            k += 1
        for p in pending:
            if p is not None:
                p.result()
        clock.io(lambda: (f.flush(), os.fsync(f.fileno())))
    os.replace(tmp, path)
    _fsync_dir(os.path.dirname(os.path.abspath(path)))
    if timings is not None:
        timings.update(total_s=time.perf_counter() - t0, bytes=h.file_bytes())
    return h


def _fsync_dir(d):
    try:
        fd = os.open(d, os.O_RDONLY)
    except OSError:
        return
    try:
        os.fsync(fd)
    except OSError:
        pass
    finally:
        os.close(fd)


def read_checked(path, sizes: tuple, alpha: float, world: int | None = None):
    """(header, episode table) of the snapshot at `path`, refused (ValueError) unless the shard can take it."""
    with open(path, "rb") as f:
        h = Header.read(f)
        check_header(h, path, sizes, alpha, world)
        return h, read_episodes(f, h)


def load(dev, path, world: int | None = None, restore_rng: bool = True, stage_bytes: int = STAGE_BYTES,
         timings: dict | None = None) -> dict:
    """Restores the snapshot at `path` into the EMPTY DeviceReplay `dev` (checked in full before the shard is touched;
    a refusal during the restore leaves the shard empty).  With restore_rng the device's default CUDA generator gets the
    saved state back.  Returns the header's fields plus `dropped`, the episodes a smaller ring could not hold."""
    import torch

    from . import native as nv
    t0 = time.perf_counter()
    clock = _Clock(timings)
    c = dev.cfg
    h, table = read_checked(path, (c.obs, c.act, c.hidden, c.burn_in, c.learning, c.n_step), c.priority_exponent, world)
    lib, hd = dev.lib, dev._h
    info = nv.ReplaySnapshotInfo(**{k: getattr(h, k) for k, _ in nv.ReplaySnapshotInfo._fields_})
    cols = [np.ascontiguousarray(table[k]) for k in ("row_start", "n_rows", "n_starts", "serial")]
    P = lambda a: a.ctypes.data_as(c_void_p)  # noqa: E731
    dropped = c_longlong(0)
    stream = nv.current_stream()
    nv.check(lib.r2d2_replay_import_begin(hd, byref(info), *[P(a) for a in cols], byref(dropped), stream))
    rb = h.row_bytes()
    begun = True
    try:
        bufs = [_pinned(min(h.chunk_rows, max(h.rows_used, 1)) * rb) for _ in range(2)]
        with open(path, "rb") as f, ThreadPoolExecutor(max_workers=1) as pool:
            f.seek(h.header_bytes + h.n_episodes * _EPISODE.itemsize)

            def read_into(buf, n):
                got = clock.io(lambda: f.readinto(memoryview(buf.numpy())[:n]))
                if got != n:
                    raise ValueError("replay snapshot %s: truncated rows" % path)

            chunks = [(p, min(h.chunk_rows, h.rows_used - p)) for p in range(0, h.rows_used, h.chunk_rows)]
            nxt = pool.submit(read_into, bufs[0], chunks[0][1] * rb) if chunks else None
            for k, (first, n) in enumerate(chunks):
                nxt.result()
                if k + 1 < len(chunks):          # read the next chunk while this one goes to the device
                    nxt = pool.submit(read_into, bufs[(k + 1) % 2], chunks[k + 1][1] * rb)
                base = bufs[k % 2].data_ptr()
                ptrs = [c_void_p(base + off) for off, _ in _chunk_layout(h, n)]
                clock.device("device_s", lambda: nv.check(lib.r2d2_replay_import_rows(hd, first, n, *ptrs, stream)))
        begun = False
        clock.device("rebuild_s", lambda: nv.check(lib.r2d2_replay_import_end(hd, stream)))
    except BaseException:
        if begun:                                # empty the shard: the import cannot complete
            lib.r2d2_replay_import_end(hd, stream)
        raise
    if restore_rng:
        torch.cuda.set_rng_state(torch.frombuffer(bytearray(h.rng_state), dtype=torch.uint8), dev.device)
    if timings is not None:
        timings.update(total_s=time.perf_counter() - t0, bytes=h.file_bytes())
    out = {f.name: getattr(h, f.name) for f in fields(h)}
    out["dropped"] = int(dropped.value)
    return out

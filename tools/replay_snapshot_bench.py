"""Replay snapshot save / restore time (DeviceReplay.save_snapshot / load_snapshot) at cfg-3 and cfg-2 shapes, in both
state storage types, for a shard of several GB, in one process on one GPU.

Per case the shard is filled with cfg-3-sized actor files (16 episodes of 250 + 5 rows) to about --gb GB of live rows,
written to a temporary local directory (deleted afterwards) and restored into a fresh shard of the same capacity.
Reported: the whole save / restore (host clock), the device copies (CUDA events around the export / import calls), the
file I/O (host clock, summed over the writer / reader thread's calls; they overlap the copies) and the restore's tree
rebuild (CUDA events).  The restore reads a file the save has just written, so it is normally served from the page
cache: its I/O share is a lower bound for a cold read.  The card's name and power limit are read in the same process.
Prints one JSON line; --out writes it too.

    python tools/replay_snapshot_bench.py [--gb 3] [--out bench_out/replay_snapshot.json]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "pytorch-r2d2-dpg_b200")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from r2d2_b200 import engine  # noqa: E402

CONFIGS = {"cfg3": dict(obs=376, act=17, hidden=512, batch=512, burn_in=40, learning=80, n_step=5),
           "cfg2": dict(obs=17, act=6, hidden=256, batch=256, burn_in=40, learning=80, n_step=5)}
EPISODE_ROWS = 250


def card():
    q = "name,power.limit"
    try:
        line = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i",
                               str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(","), (s.strip() for s in line.strip().split(","))))
    except (OSError, subprocess.SubprocessError):
        return {"name": torch.cuda.get_device_name()}


def actor_file(cfg, rng, n_eps=16):
    eps = []
    for _ in range(n_eps):
        n = EPISODE_ROWS + cfg.n_step
        term = np.zeros(n, np.float32)
        term[EPISODE_ROWS:] = 1
        st = np.empty((EPISODE_ROWS, 4, 2, cfg.hidden), np.float32)
        st[:, :, 0] = np.tanh(rng.standard_normal((EPISODE_ROWS, 4, cfg.hidden), dtype=np.float32))
        st[:, :, 1] = 2 * rng.standard_normal((EPISODE_ROWS, 4, cfg.hidden), dtype=np.float32)
        eps.append((rng.standard_normal((n, cfg.obs), dtype=np.float32), rng.uniform(-1, 1, (n, cfg.act)).astype(np.float32),
                    rng.standard_normal(n, dtype=np.float32), term, st,
                    rng.uniform(0.01, 1, EPISODE_ROWS - cfg.burn_in - cfg.learning).astype(np.float32)))
    return eps


def case(name, dtype, gb, tmp):
    cfg = engine.PathConfig(**CONFIGS[name], replay_state_dtype=dtype, priority_exponent=0.9)
    row = 4 * (cfg.obs + cfg.act + 3) + (16 if dtype == "float16" else 32) * cfg.hidden
    rows = int(gb * 1e9 / row)
    cap = rows + 4096
    rng = np.random.default_rng(0)
    files = [actor_file(cfg, rng) for _ in range(2)]
    src = engine.DeviceReplay(cfg, capacity_rows=cap)
    k = 0
    while src.snapshot_info()["rows_used"] + 16 * (EPISODE_ROWS + cfg.n_step) <= cap:
        src.add_episodes(files[k % 2])
        k += 1
    torch.cuda.synchronize()
    path = os.path.join(tmp, "shard")
    ts, tl = {}, {}
    src.save_snapshot(path, timings=ts)
    dst = engine.DeviceReplay(cfg, capacity_rows=cap)
    dst.load_snapshot(path, timings=tl)
    torch.cuda.synchronize()
    same = all(src.tree_level(l).equal(dst.tree_level(l)) for l in range(int(src.stats()["tree_levels"])))
    info = src.snapshot_info()
    src.close()
    dst.close()
    os.remove(path)
    r = lambda d: {k: round(v, 4) for k, v in d.items() if k.endswith("_s")}  # noqa: E731
    return {"config": name, "state_dtype": dtype, "rows": int(info["rows_used"]), "episodes": int(info["n_episodes"]),
            "file_GB": round(ts["bytes"] / 1e9, 3), "save": r(ts), "restore": r(tl),
            "save_GB_per_s": round(ts["bytes"] / 1e9 / ts["total_s"], 2),
            "restore_GB_per_s": round(tl["bytes"] / 1e9 / tl["total_s"], 2), "tree_identical": bool(same)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gb", type=float, default=3.0, help="live rows per shard, GB")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    tmp = tempfile.mkdtemp(prefix="replay_snapshot_bench_")
    try:
        res = {"card": card(), "gb": a.gb, "cases": [case(n, d, a.gb, tmp) for n in CONFIGS for d in ("float32", "float16")]}
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

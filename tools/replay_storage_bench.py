"""Replay shard, fp32 vs fp16 recurrent-state storage (PathConfig.replay_state_dtype), in one process on one GPU.

The two modes alternate over 3 rounds.  Reported per mode:
  - the gather kernel per sample_into (r2d2_replay_gather at the drawn leaves into the engine's batch), CUDA events;
  - sample_into (tree draw + gather), CUDA events;
  - the replay-fed pipelined learner iteration (step + write-back + next draw in the prefetch hook), CUDA events;
    at cfg-3 (obs 376, act 17, H 512, batch 512) and cfg-2 (obs 17, act 6, H 256, batch 256), window 40 + 80 + 5;
  - add_episodes of one cfg-3-sized actor file (16 episodes of 250 + 5 rows), host clock, median of 9;
  - the ring rows that fit a fixed device-memory budget, from device_bytes().
The card's name, power limit and SM clocks are read in the same process.  Prints one JSON line; --out writes it too.

    python tools/replay_storage_bench.py [--rounds 3] [--steps 10] [--out bench_out/replay_storage.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "pytorch-r2d2-dpg_b200")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from r2d2_b200 import engine  # noqa: E402
from r2d2_b200 import native as nv  # noqa: E402

CONFIGS = {"cfg3": dict(obs=376, act=17, hidden=512, batch=512, burn_in=40, learning=80, n_step=5),
           "cfg2": dict(obs=17, act=6, hidden=256, batch=256, burn_in=40, learning=80, n_step=5)}
MODES = ("float32", "float16")
EPISODE_ROWS = 250          # env steps per episode; + n_step pad rows
BUDGET = 40 * 10 ** 9       # device bytes for the ring-capacity comparison


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
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


def events_ms(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


class Setup:
    """One shard of 4 actor files and one engine for a config and a storage mode."""

    def __init__(self, name, mode, files):
        self.cfg = engine.PathConfig(**CONFIGS[name], replay_state_dtype=mode)
        rows = sum(e[0].shape[0] for f in files for e in f)
        self.rp = engine.DeviceReplay(self.cfg, capacity_rows=rows)
        for f in files:
            self.rp.add_episodes(f)
        self.eng = engine.LearnerEngine(self.cfg, seed=1)
        self.gen = torch.Generator(device="cuda").manual_seed(0)
        self.rp.sample_into(self.eng, generator=self.gen)
        torch.cuda.synchronize()

    def gather(self):
        e = self.eng
        nv.check(self.rp.lib.r2d2_replay_gather(self.rp._h, nv.dptr(e.leaf_idx, torch.int64), self.cfg.batch,
                                                nv.dptr(e.obs), nv.dptr(e.act), nv.dptr(e.rew), nv.dptr(e.term),
                                                nv.dptr(e.states), nv.current_stream()))

    def sample(self):
        self.rp.sample_into(self.eng, generator=self.gen)

    def step(self):
        def hook(e, used):
            self.rp.update_priorities(used.leaf_idx, used.priority)
            self.rp.sample_into(e, generator=self.gen)
        self.eng.step(prefetch=hook)

    def close(self):
        self.eng.close()
        self.rp.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("replay_storage_bench needs a CUDA device")
    rng = np.random.default_rng(0)
    out = {"card": card(), "rounds": args.rounds, "steps": args.steps}
    res = {}
    for name in CONFIGS:
        files = [actor_file(engine.PathConfig(**CONFIGS[name]), rng) for _ in range(4)]
        for rnd in range(args.rounds):
            for mode in (MODES if rnd % 2 == 0 else MODES[::-1]):
                s = Setup(name, mode, files)
                for _ in range(3):
                    s.gather()
                    s.sample()
                r = res.setdefault(f"{name}/{mode}", {"gather_us": [], "sample_into_us": [], "iteration_ms": []})
                r["gather_us"].append(1e3 * events_ms(s.gather, 200))
                r["sample_into_us"].append(1e3 * events_ms(s.sample, 200))
                for _ in range(3):
                    s.step()
                r["iteration_ms"].append(events_ms(s.step, args.steps))
                s.close()
    # ingest: one cfg-3 actor file into a shard that holds it 8 times
    c3 = engine.PathConfig(**CONFIGS["cfg3"])
    f = actor_file(c3, rng)
    rows = sum(e[0].shape[0] for e in f)
    for rnd in range(args.rounds):
        for mode in (MODES if rnd % 2 == 0 else MODES[::-1]):
            rp = engine.DeviceReplay(engine.PathConfig(**CONFIGS["cfg3"], replay_state_dtype=mode), capacity_rows=8 * rows)
            rp.add_episodes(f)                                   # warm: staging allocated, modules loaded
            ts = []
            for _ in range(9):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                rp.add_episodes(f)                               # synchronises before it returns
                ts.append(1e3 * (time.perf_counter() - t0))
            res.setdefault(f"cfg3/{mode}", {}).setdefault("add_episodes_ms", []).append(float(np.median(ts)))
            rp.close()
    # ring rows in a fixed budget: marginal bytes per row from two capacities, the staging of one file on top
    for name in CONFIGS:
        for mode in MODES:
            cfg = engine.PathConfig(**CONFIGS[name], replay_state_dtype=mode)
            sizes = []
            for cap in (200_000, 400_000):
                rp = engine.DeviceReplay(cfg, capacity_rows=cap)
                if cap == 200_000:
                    b0 = rp.device_bytes()
                    rp.add_episodes(actor_file(cfg, rng))
                    staging = rp.device_bytes() - b0
                sizes.append(rp.device_bytes() - (staging if cap == 200_000 else 0))
                rp.close()
            per_row = (sizes[1] - sizes[0]) / 200_000
            r = res.setdefault(f"{name}/{mode}", {})
            r["device_bytes_per_row"] = round(per_row, 2)
            r["staging_bytes_one_file"] = int(staging)
            r["rows_in_budget"] = int((BUDGET - staging - (sizes[0] - per_row * 200_000)) // per_row)
    for k, r in res.items():
        for m in [m for m in r if isinstance(r[m], list)]:
            v = r[m]
            r[m] = {"median": round(float(np.median(v)), 3), "min": round(float(min(v)), 3),
                    "max": round(float(max(v)), 3)}
    out["budget_bytes"] = BUDGET
    out["results"] = res
    for name in CONFIGS:
        out[f"{name}_rows_ratio_f16_over_f32"] = round(res[f"{name}/float16"]["rows_in_budget"]
                                                       / res[f"{name}/float32"]["rows_in_budget"], 3)
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()

"""Replay shard, recurrent states in HBM vs in pinned host memory (PathConfig.replay_state_memory), one process, one GPU.

The card's name, power limit and current PCIe link (nvidia-smi, queries only) and the host's MemAvailable are read in the
same run.  The device-state and host-state arms alternate over --rounds rounds, in fp32 and fp16 state storage.
Reported per arm:
  - the gather kernel per sample_into (r2d2_replay_gather at the drawn leaves into the engine's batch), CUDA events over
    --gathers calls, and the host-read rate it implies: the batch's state bytes (8 B H x 4 or 2) over that time;
  - the replay-fed pipelined learner iteration (step + write-back + next draw in the prefetch hook), CUDA events over
    --steps steps, as in tools/replay_storage_bench.py;
    at cfg-3 (obs 376, act 17, H 512, batch 512) and cfg-2 (obs 17, act 6, H 256, batch 256), window 40 + 80 + 5;
  - add_episodes of one cfg-3 actor file (16 episodes of 250 + 5 rows), host clock, median of 9;
  - shard creation time, host_bytes() and device_bytes() of a ring sized to --host-gb of fp32 cfg-3 states.
Prints one JSON line; --out writes it too.

    python tools/replay_host_states_bench.py [--rounds 3] [--steps 10] [--gathers 200] [--host-gb 2]
                                            [--out bench_out/replay_host_states.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "pytorch-r2d2-dpg_b200"), os.path.join(ROOT, "tools")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from r2d2_b200 import engine  # noqa: E402
from replay_storage_bench import CONFIGS, Setup, actor_file, events_ms  # noqa: E402

MEMORIES = ("device", "host")
DTYPES = ("float32", "float16")


def card():
    q = "name,power.limit,pcie.link.gen.current,pcie.link.width.current,pcie.link.gen.max,pcie.link.width.max"
    try:
        line = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i",
                               str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        out = dict(zip(q.split(","), (s.strip() for s in line.strip().split(","))))
    except (OSError, subprocess.SubprocessError):
        out = {"name": torch.cuda.get_device_name()}
    try:
        with open("/proc/meminfo") as f:
            for ln in f:
                if ln.startswith("MemAvailable:"):
                    out["host_mem_available_gb"] = round(int(ln.split()[1]) * 1024 / 1e9, 1)
    except OSError:
        pass
    return out


class TierSetup(Setup):
    def __init__(self, name, memory, dtype, files):
        self.cfg = engine.PathConfig(**CONFIGS[name], replay_state_dtype=dtype, replay_state_memory=memory)
        rows = sum(e[0].shape[0] for f in files for e in f)
        self.rp = engine.DeviceReplay(self.cfg, capacity_rows=rows)
        for f in files:
            self.rp.add_episodes(f)
        self.eng = engine.LearnerEngine(self.cfg, seed=1)
        self.gen = torch.Generator(device="cuda").manual_seed(0)
        self.rp.sample_into(self.eng, generator=self.gen)
        torch.cuda.synchronize()


def arms(rnd):
    out = [(m, d) for d in DTYPES for m in MEMORIES]
    return out if rnd % 2 == 0 else out[::-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--gathers", type=int, default=200)
    ap.add_argument("--host-gb", type=float, default=2.0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("replay_host_states_bench needs a CUDA device")
    rng = np.random.default_rng(0)
    out = {"card": card(), "rounds": args.rounds, "steps": args.steps, "gathers": args.gathers}
    res = {}
    for name in CONFIGS:
        files = [actor_file(engine.PathConfig(**CONFIGS[name]), rng) for _ in range(4)]
        for rnd in range(args.rounds):
            for memory, dtype in arms(rnd):
                s = TierSetup(name, memory, dtype, files)
                for _ in range(3):
                    s.gather()
                    s.step()
                r = res.setdefault(f"{name}/{memory}/{dtype}", {"gather_us": [], "iteration_ms": []})
                r["gather_us"].append(1e3 * events_ms(s.gather, args.gathers))
                r["iteration_ms"].append(events_ms(s.step, args.steps))
                s.close()
    c3 = CONFIGS["cfg3"]
    f = actor_file(engine.PathConfig(**c3), rng)
    rows = sum(e[0].shape[0] for e in f)
    for rnd in range(args.rounds):
        for memory, dtype in arms(rnd):
            rp = engine.DeviceReplay(engine.PathConfig(**c3, replay_state_dtype=dtype, replay_state_memory=memory),
                                     capacity_rows=8 * rows)
            rp.add_episodes(f)                                   # warm: staging allocated, modules loaded
            ts = []
            for _ in range(9):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                rp.add_episodes(f)                               # synchronises before it returns
                ts.append(1e3 * (time.perf_counter() - t0))
            res.setdefault(f"cfg3/{memory}/{dtype}", {}).setdefault("add_episodes_ms", []).append(float(np.median(ts)))
            rp.close()
    for k, r in res.items():
        for m in [m for m in r if isinstance(r[m], list)]:
            v = r[m]
            r[m] = {"median": round(float(np.median(v)), 3), "min": round(float(min(v)), 3),
                    "max": round(float(max(v)), 3)}
        name, memory, dtype = k.split("/")
        c = CONFIGS[name]
        state_bytes = 8 * c["batch"] * c["hidden"] * (2 if dtype == "float16" else 4)
        r["state_bytes_per_batch"] = state_bytes
        if memory == "host" and "gather_us" in r:
            r["host_read_gb_per_s"] = round(state_bytes / (r["gather_us"]["median"] * 1e-6) / 1e9, 2)
    # creation at the --host-gb budget (fp32 cfg-3 states: 16 KB per row)
    cfg = engine.PathConfig(**c3, replay_state_memory="host")
    cap = int(args.host_gb * 1e9 / (32 * c3["hidden"]))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    rp = engine.DeviceReplay(cfg, capacity_rows=cap)
    torch.cuda.synchronize()
    out["create"] = {"host_gb": args.host_gb, "capacity_rows": cap, "seconds": round(time.perf_counter() - t0, 3),
                     "host_bytes": rp.host_bytes(), "device_bytes": rp.device_bytes()}
    rp.close()
    out["results"] = res
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()

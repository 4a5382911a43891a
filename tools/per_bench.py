"""Cost of prioritized replay (priority exponent alpha, importance-sampling exponent beta) on the learner's hot path.

  python tools/per_bench.py [--steps 30] [--rounds 3]

1. Replay-fed pipelined learner iterations (bench.py's HBM-resident loop: write-back, draw + gather, LearnerEngine.step)
   at cfg-3 and cfg-2, (alpha, beta) = (1, 0) - the default, unweighted kernels - against (0.9, 0.6), published R2D2's
   values.  The two arms alternate `--rounds` times in one process, so drift of clocks or of other work on the host
   shows up as spread rather than as a difference.
2. r2d2_replay_add_episodes for one cfg-3-sized actor file (16 episodes of 250 steps) at alpha = 1 and alpha = 0.9.

Prints one JSON line with the card's name, power limit and SM clock beside the numbers.
"""
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "pytorch-r2d2-dpg_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402

ARMS = {"default": dict(priority_exponent=1.0, is_exponent=0.0), "per": dict(priority_exponent=0.9, is_exponent=0.6)}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except Exception as e:  # noqa: BLE001
        return {"error": repr(e)}


def iterations(name, episodes, steps, rounds, dev):
    from r2d2_b200 import engine
    c = bench.CONFIGS[name]
    arms = {k: bench.Arm(engine, dict(c, **v), dev, 0, episodes, data_parallel=False) for k, v in ARMS.items()}
    ms = {k: [] for k in arms}
    for _ in range(rounds):
        for k, arm in arms.items():
            ms[k].append(arm.time_resident(steps, 5, torch.cuda.synchronize))
    launches = {k: arm.launches_per_step + (1 if arm.eng.importance_weighting else 0) for k, arm in arms.items()}
    for arm in arms.values():
        arm.close()
    med = {k: statistics.median(v) for k, v in ms.items()}
    return {"workload": bench.workload_string(name, c), "ms_per_step": ms, "median_ms": med,
            "overhead_pct": 100.0 * (med["per"] / med["default"] - 1.0), "gpu_launches_per_step": launches}


def ingest(dev, rounds):
    from r2d2_b200 import engine
    c = bench.CONFIGS["cfg3"]
    E, n_eps = 250, 16
    n_rows = E + c["n_step"]
    rng = np.random.default_rng(3)
    eps = []
    for _ in range(n_eps):
        term = np.zeros(n_rows, np.float32)
        term[E:] = 1
        eps.append((rng.standard_normal((n_rows, c["obs"]), dtype=np.float32),
                    rng.uniform(-1, 1, (n_rows, c["act"])).astype(np.float32),
                    rng.standard_normal(n_rows, dtype=np.float32), term,
                    0.1 * rng.standard_normal((E, 4, 2, c["hidden"]), dtype=np.float32),
                    rng.uniform(0.01, 1.0, E - (c["burn_in"] + c["learning"])).astype(np.float32)))
    shards = {k: engine.DeviceReplay(engine.PathConfig(**c, priority_exponent=v["priority_exponent"]),
                                     capacity_rows=4 * n_eps * n_rows, device=dev) for k, v in ARMS.items()}
    for rp in shards.values():
        rp.add_episodes(eps)                                          # warm-up (module load, first copies)
    ms = {k: [] for k in shards}
    for _ in range(rounds * 3):
        for k, rp in shards.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            rp.add_episodes(eps)                                      # synchronises its stream before returning
            ms[k].append(1e3 * (time.perf_counter() - t0))
    for rp in shards.values():
        rp.close()
    med = {k: statistics.median(v) for k, v in ms.items()}
    return {"file": f"{n_eps} episodes x {n_rows} rows at cfg-3 widths", "ms_per_call": ms, "median_ms": med,
            "overhead_pct": 100.0 * (med["per"] / med["default"] - 1.0)}


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("per_bench.py needs a CUDA device")
    torch.cuda.set_device(0)
    dev = torch.device("cuda:0")
    before = card()
    out = {"arms": ARMS, "card_before": before,
           "cfg3": iterations("cfg3", 256, args.steps, args.rounds, dev),
           "cfg2": iterations("cfg2", 128, args.steps, args.rounds, dev),
           "add_episodes": ingest(dev, args.rounds), "card_after": card()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()

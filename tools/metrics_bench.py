"""Cost of the learner metrics (R2D2_METRICS, csrc/metrics.cu) on the learner's hot path.

  python tools/metrics_bench.py [--steps 30] [--rounds 3]

1. Replay-fed pipelined learner iterations (bench.py's HBM-resident loop: write-back, draw + gather, LearnerEngine.step)
   at cfg-3 and cfg-2, metrics off and on, alternated `--rounds` times in one process: medians and ranges.
2. Device time per launch of metrics_critic_kernel, metrics_actor_kernel and the norm kernel that metrics add before
   each Adam (grad_norm_kernel; no clipping here), from torch.profiler over a few steps of the "on" arm in a separate,
   untimed run.
3. Host time of one LearnerMetrics.read() at a log point: the read right after 100 issued steps (it waits for the
   stream to drain, as the drop-in learner's read does), and a read of 100 records on an idle stream (the copy and the
   synchronisation alone).

Prints one JSON line with the card's name, power limit and SM clock beside the numbers.
"""
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "pytorch-r2d2-dpg_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

import bench  # noqa: E402
from optim_bench import card  # noqa: E402

ARMS = {"off": dict(), "on": dict(metrics=True)}
KERNELS = ("metrics_critic_kernel", "metrics_actor_kernel", "grad_norm_kernel")


def kernel_times(arm, steps):
    from torch.profiler import ProfilerActivity, profile
    arm.eng.discard_prefetched()
    arm.rp.sample_into(arm.eng, generator=arm.gen)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            arm.step_resident()
        torch.cuda.synchronize()
    agg = {}
    for e in prof.events():
        for k in KERNELS:
            if k in e.name:
                t = agg.setdefault(k, [0.0, 0])
                t[0] += e.device_time if hasattr(e, "device_time") else e.cuda_time
                t[1] += 1
    return {k: {"us_per_launch": v[0] / v[1], "launches_per_step": v[1] / steps} for k, v in sorted(agg.items())}


def read_times(arm):
    m = arm.eng.metrics
    arm.eng.discard_prefetched()
    arm.rp.sample_into(arm.eng, generator=arm.gen)
    torch.cuda.synchronize()
    m.read()
    out = {}
    for mode in ("after_issue", "idle"):
        ms = []
        for _ in range(3):
            for _ in range(100):
                arm.step_resident()
            if mode == "idle":
                torch.cuda.synchronize()
            t0 = time.perf_counter()
            rec = m.read()
            ms.append(1e3 * (time.perf_counter() - t0))
            assert len(rec["iteration"]) >= 99
        out[mode] = {"ms": ms, "median_ms": statistics.median(ms)}
    return out


def iterations(name, episodes, steps, rounds, dev):
    from r2d2_b200 import engine
    c = bench.CONFIGS[name]
    arms = {k: bench.Arm(engine, dict(c, **v), dev, 0, episodes, data_parallel=False) for k, v in ARMS.items()}
    ms = {k: [] for k in arms}
    for _ in range(rounds):
        for k, arm in arms.items():
            ms[k].append(arm.time_resident(steps, 5, torch.cuda.synchronize))
            if arm.eng.metrics is not None:
                arm.eng.metrics.read()          # the timed window never overruns the ring
    launches = {k: arm.launches_per_step for k, arm in arms.items()}
    kernels = kernel_times(arms["on"], 5)
    arms["on"].eng.metrics.read()
    reads = read_times(arms["on"])
    cf = arms["on"].cfg
    for arm in arms.values():
        arm.close()
    med = {k: statistics.median(v) for k, v in ms.items()}
    lba = cf.learning * cf.batch * cf.act
    return {"workload": bench.workload_string(name, c), "ms_per_step": ms, "median_ms": med,
            "range_ms": {k: [min(v), max(v)] for k, v in ms.items()},
            "overhead_pct": 100.0 * (med["on"] / med["off"] - 1.0), "gpu_launches_per_step": launches,
            "critic_kernel_bytes_read": 4 * (2 * lba + 2 * cf.batch), "kernels": kernels, "read": reads}


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("metrics_bench.py needs a CUDA device")
    torch.cuda.set_device(0)
    dev = torch.device("cuda:0")
    out = {"card_before": card(),
           "cfg3": iterations("cfg3", 256, args.steps, args.rounds, dev),
           "cfg2": iterations("cfg2", 128, args.steps, args.rounds, dev), "card_after": card()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()

"""Device time per kernel inside real learner iterations (dev tool).

Runs the bench.py workload (HBM-resident replay shard, sample -> learner step -> priority write-back) for a few warm-up
iterations, then profiles --steps iterations with torch.profiler (CUDA activity only) and adds up the device time of
every kernel, per instantiation and per kernel name.  Shares are of the summed kernel time, which is close to the
iteration time because the hot path is one stream of back-to-back launches.

  python tools/kernel_breakdown.py OUT_DIR [--config cfg3] [--steps 5] [--warmup 5]

writes OUT_DIR/kernel_breakdown_<config>.json and prints the top entries.
"""
import argparse
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "pytorch-r2d2-dpg_b200")]

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import bench  # noqa: E402
from r2d2_b200 import engine  # noqa: E402


def short_name(name):
    """'void r2d2::(anonymous namespace)::lstm_scan_bwd_kernel<512, 16>(r2d2::ScanBwdParams)' ->
    'lstm_scan_bwd_kernel<512, 16>' (memcpy / memset records keep their names)."""
    if name.startswith(("Memcpy", "Memset")):
        return name
    name = re.sub(r"(\w+::|\(anonymous namespace\)::)+", "", re.sub(r"^void ", "", name))
    depth = 0
    for i, ch in enumerate(name):   # the parameter list is the first '(' outside the template arguments
        depth += (ch == "<") - (ch == ">")
        if ch == "(" and depth == 0:
            return name[:i].strip()
    return name.strip()


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), f"--query-gpu={q}",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), (v.strip() for v in out.split(","))))
    except (OSError, subprocess.SubprocessError):
        return {"name": torch.cuda.get_device_name()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--config", default="cfg3", choices=sorted(bench.CONFIGS))
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--episodes", type=int, default=384)
    args = ap.parse_args()

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    arm = bench.Arm(engine, bench.CONFIGS[args.config], dev, 0, args.episodes, data_parallel=True)
    ms = arm.time_resident(args.steps, args.warmup, torch.cuda.synchronize)   # unprofiled reference time
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            arm.step_resident()
        torch.cuda.synchronize()

    per_inst, per_name = {}, {}
    for ev in prof.key_averages():
        us = float(getattr(ev, "self_device_time_total", 0.0) or getattr(ev, "self_cuda_time_total", 0.0))
        if us <= 0:
            continue
        inst = short_name(ev.key)
        base = inst.split("<", 1)[0]
        for table, key in ((per_inst, inst), (per_name, base)):
            e = table.setdefault(key, {"us_per_iter": 0.0, "calls_per_iter": 0.0})
            e["us_per_iter"] += us / args.steps
            e["calls_per_iter"] += ev.count / args.steps
    total = sum(e["us_per_iter"] for e in per_inst.values())
    for table in (per_inst, per_name):
        for e in table.values():
            e["share"] = e["us_per_iter"] / total
    order = lambda t: dict(sorted(t.items(), key=lambda kv: -kv[1]["us_per_iter"]))  # noqa: E731
    result = {"config": bench.workload_string(args.config, bench.CONFIGS[args.config]), "steps": args.steps,
              "warmup": args.warmup, "ms_per_step_unprofiled": ms, "kernel_us_per_iter": total,
              "gpu": gpu_info(), "per_kernel": order(per_name), "per_instantiation": order(per_inst)}
    arm.close()
    os.makedirs(args.out_dir, exist_ok=True)
    path = os.path.join(args.out_dir, f"kernel_breakdown_{args.config}.json")
    with open(path, "w") as f:
        json.dump(result, f, indent=1)
    print(f"{args.config}: {ms:.3f} ms/iteration unprofiled, {total / 1e3:.3f} ms of kernel time per iteration")
    for k, e in list(result["per_kernel"].items())[:15]:
        print(f"  {e['us_per_iter'] / 1e3:8.3f} ms  {100 * e['share']:5.1f} %  {e['calls_per_iter']:7.1f} calls  {k}")
    print(f"wrote {path}")


if __name__ == "__main__":
    main()

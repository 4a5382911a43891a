"""Cost of the optimiser-step extras (Polyak target update, gradient-norm clipping) on the learner's hot path.

  python tools/optim_bench.py [--steps 30] [--rounds 3]

1. Replay-fed pipelined learner iterations (bench.py's HBM-resident loop: write-back, draw + gather, LearnerEngine.step)
   at cfg-3 and cfg-2 in three arms that alternate `--rounds` times in one process:
     default    target_tau 1, target_interval 500, no clipping (the reference's hard copy);
     soft       target_tau 0.005 at target_interval 1 (DDPG-style): the Polyak blend rides on both Adam launches, and
                every iteration updates the targets, so the next batch's target chains never run ahead;
     soft_clip  soft + grad_clip_norm 1e-4, small enough that both nets clip (the JSON line reports the norms).
2. The optimiser kernels alone: device time per launch of each adam_kernel instantiation and of grad_norm_kernel, taken
   from torch.profiler over a few steps of each arm in a separate, untimed run.

Prints one JSON line with the card's name, power limit and SM clock beside the numbers.
"""
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "pytorch-r2d2-dpg_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

import bench  # noqa: E402

CLIP = 1e-4
ARMS = {"default": dict(),
        "soft": dict(target_tau=0.005, target_interval=1),
        "soft_clip": dict(target_tau=0.005, target_interval=1, grad_clip_norm=CLIP)}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except Exception as e:  # noqa: BLE001
        return {"error": repr(e)}


def kernel_times(arms, steps):
    """Mean device time per launch (us) of the optimiser kernels, per arm, from a profiled run of `steps` steps."""
    from torch.profiler import ProfilerActivity, profile
    out = {}
    for k, arm in arms.items():
        arm.eng.discard_prefetched()
        arm.rp.sample_into(arm.eng, generator=arm.gen)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(steps):
                arm.step_resident()
            torch.cuda.synchronize()
        agg = {}
        for e in prof.events():
            name = e.name
            if "adam_kernel" in name or "grad_norm_kernel" in name:
                short = "grad_norm_kernel" if "grad_norm_kernel" in name else name[name.index("adam_kernel"):].split("(")[0]
                t = agg.setdefault(short, [0.0, 0])
                t[0] += e.device_time if hasattr(e, "device_time") else e.cuda_time
                t[1] += 1
        out[k] = {n: {"us_per_launch": v[0] / v[1], "launches": v[1]} for n, v in sorted(agg.items())}
    return out


def iterations(name, episodes, steps, rounds, dev):
    from r2d2_b200 import engine
    c = bench.CONFIGS[name]
    arms = {k: bench.Arm(engine, dict(c, **v), dev, 0, episodes, data_parallel=False) for k, v in ARMS.items()}
    ms = {k: [] for k in arms}
    for _ in range(rounds):
        for k, arm in arms.items():
            ms[k].append(arm.time_resident(steps, 5, torch.cuda.synchronize))
    launches = {k: arm.launches_per_step for k, arm in arms.items()}
    norms = arms["soft_clip"].eng.grad_norms.cpu().tolist()
    kernels = kernel_times(arms, 5)
    n_params = {n: arms["default"].eng.flat[n].numel() for n in ("critic", "actor")}
    for arm in arms.values():
        arm.close()
    med = {k: statistics.median(v) for k, v in ms.items()}
    return {"workload": bench.workload_string(name, c), "params": n_params, "ms_per_step": ms, "median_ms": med,
            "overhead_pct": {k: 100.0 * (med[k] / med["default"] - 1.0) for k in ("soft", "soft_clip")},
            "gpu_launches_per_step": launches, "soft_clip_grad_norms": {"critic": norms[0], "actor": norms[1],
                                                                       "clip": CLIP}, "kernels": kernels}


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("optim_bench.py needs a CUDA device")
    torch.cuda.set_device(0)
    dev = torch.device("cuda:0")
    out = {"arms": ARMS, "card_before": card(),
           "cfg3": iterations("cfg3", 256, args.steps, args.rounds, dev),
           "cfg2": iterations("cfg2", 128, args.steps, args.rounds, dev), "card_after": card()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()

"""Cost of TD3's target (twin critic, target policy smoothing) on the learner path.

  python tools/td3_bench.py [--steps 20] [--rounds 3] [--reps 50]

1. Replay-fed pipelined learner iterations (bench.py's HBM-resident loop) at cfg-3 and cfg-2: the defaults, the twin
   critic, and the twin with smoothing (sigma 0.2, c 0.5).  The arms alternate `--rounds` times in one process, so drift
   of clocks or of other work on the host shows up as spread rather than as a difference.  Launches per iteration and
   the arena bytes the twin adds (from the library's ChainWs::floats) are reported per arm.
2. The smoothing kernel and the clipped double-Q minimum alone, at each config's L x B x A: GPU time per call from
   torch.profiler's kernel records, median over `--reps` calls, in a separate run.

Prints one JSON line with the card's name, power limit and SM clock beside the numbers.
"""
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "pytorch-r2d2-dpg_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from per_bench import card  # noqa: E402

ARMS = {"default": {}, "twin": dict(twin_critic=True),
        "twin_smooth": dict(twin_critic=True, target_noise=0.2, target_noise_clip=0.5)}


def kernels(name, reps):
    """The smoothing kernel through its C entry; the minimum inside one twin iteration (it has no entry of its own)."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    from r2d2_b200 import native as nv
    c = bench.CONFIGS[name]
    n = c["learning"] * c["batch"] * c["act"]
    mu = torch.rand(n, device="cuda") * 2 - 1
    out = torch.empty_like(mu)

    def call(it):
        nv.check(nv.lib().r2d2_target_smoothing(nv.dptr(mu), nv.dptr(out), n, 0.2, 0.5, 0, 0, it, nv.current_stream()))
    for i in range(10):
        call(i)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(reps):
            call(i)
        torch.cuda.synchronize()
    sm = [e.device_time for e in prof.events() if e.device_type == DeviceType.CUDA and "target_smoothing" in e.name]
    from r2d2_b200 import engine
    arm = bench.Arm(engine, dict(c, **ARMS["twin_smooth"]), torch.device("cuda:0"), 0, 64, data_parallel=False)
    arm.time_resident(3, 2, torch.cuda.synchronize)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        arm.time_resident(min(reps, 10), 0, torch.cuda.synchronize)
    qm = [e.device_time for e in prof.events() if e.device_type == DeviceType.CUDA and "q_min_kernel" in e.name]
    arm.close()
    return {"elements": n, "smoothing_us": statistics.median(sm) if sm else None, "smoothing_calls": len(sm),
            "q_min_us": statistics.median(qm) if qm else None, "q_min_calls": len(qm)}


def iterations(name, episodes, steps, rounds, dev):
    from r2d2_b200 import engine
    c = bench.CONFIGS[name]
    arms = {k: bench.Arm(engine, dict(c, **v), dev, 0, episodes, data_parallel=False) for k, v in ARMS.items()}
    ms = {k: [] for k in arms}
    for _ in range(rounds):
        for k, arm in arms.items():
            ms[k].append(arm.time_resident(steps, 5, torch.cuda.synchronize))
    launches = {k: arm.launches_per_step for k, arm in arms.items()}
    added = {k: arm.eng.twin_added_bytes for k, arm in arms.items()}
    for arm in arms.values():
        arm.close()
    med = {k: statistics.median(v) for k, v in ms.items()}
    rng = {k: [min(v), max(v)] for k, v in ms.items()}
    return {"workload": bench.workload_string(name, c), "ms_per_step": ms, "median_ms": med, "range_ms": rng,
            "overhead_pct": {k: 100.0 * (med[k] / med["default"] - 1.0) for k in med},
            "gpu_launches_per_step": launches, "twin_added_bytes": added}


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--kernels-only", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("td3_bench.py needs a CUDA device")
    torch.cuda.set_device(0)
    dev = torch.device("cuda:0")
    np.random.seed(0)
    out = {"arms": ARMS, "card_before": card()}
    if args.kernels_only:
        out.update(kernels_cfg3=kernels("cfg3", args.reps), kernels_cfg2=kernels("cfg2", args.reps))
    else:
        out.update(cfg3=iterations("cfg3", 256, args.steps, args.rounds, dev),
                   cfg2=iterations("cfg2", 128, args.steps, args.rounds, dev))
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

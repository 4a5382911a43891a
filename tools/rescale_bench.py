"""Cost of R2D2's n-step target options (invertible value rescaling, absolute-TD-error priorities) on the learner path.

  python tools/rescale_bench.py [--steps 30] [--rounds 3] [--reps 50]

1. The TD kernel pair alone (td_elem_kernel + td_reduce_kernel, r2d2_td_priority_ex) at cfg-3 and cfg-2 shapes, in each
   mode x metric: GPU time per call from torch.profiler's kernel records, median over `--reps` calls.
2. Replay-fed pipelined learner iterations (bench.py's HBM-resident loop) at cfg-3 and cfg-2, the default options against
   (invertible, eps 1e-3, abs).  The two arms alternate `--rounds` times in one process, so drift of clocks or of other
   work on the host shows up as spread rather than as a difference.

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

MODES = [(r, m) for r in ("reference", "invertible") for m in ("squared", "abs")]
ARMS = {"default": {}, "r2d2": dict(value_rescaling="invertible", rescaling_eps=1e-3, priority_metric="abs")}


def td_kernels(name, reps):
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    from r2d2_b200 import native as nv
    from r2d2_b200 import td_options
    c = bench.CONFIGS[name]
    L, B, A, Bn, n = c["learning"], c["batch"], c["act"], c["burn_in"], c["n_step"]
    T = Bn + L + n
    g = torch.Generator(device="cuda").manual_seed(0)
    q, qn = (torch.randn((L, B, A), device="cuda", generator=g) for _ in range(2))
    rew = torch.randn((T, B), device="cuda", generator=g)
    term = (torch.rand((T, B), device="cuda", generator=g) < 0.02).float()
    y, dq = torch.empty_like(q), torch.empty_like(q)
    td, prio, loss = torch.empty((L, B), device="cuda"), torch.empty(B, device="cuda"), torch.empty(1, device="cuda")
    P = nv.dptr
    out = {}
    for r, m in MODES:
        opts = nv.TdOptions(*td_options.TdOptions(r, 1e-3, m).native())

        def call():
            nv.check(nv.lib().r2d2_td_priority_ex(P(q), P(qn), P(rew), P(term), None, L, B, A, Bn, n, 0.997, 0.9, P(y),
                                                  P(dq), P(td), P(prio), P(loss), nv.byref(opts), nv.current_stream()))
        for _ in range(10):
            call()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                call()
            torch.cuda.synchronize()
        per = {}
        for e in prof.events():
            if e.device_type == DeviceType.CUDA and ("td_elem_kernel" in e.name or "td_reduce_kernel" in e.name):
                k = "elem" if "td_elem_kernel" in e.name else "reduce"
                per.setdefault(k, []).append(e.device_time)
        out[f"{r}/{m}"] = {k: {"median_us": statistics.median(v), "calls": len(v)} for k, v in per.items()}
        out[f"{r}/{m}"]["pair_us"] = sum(v["median_us"] for v in out[f"{r}/{m}"].values())
    return {"workload": f"L={L} B={B} A={A} (L*B*A = {L * B * A})", "kernels": out}


def iterations(name, episodes, steps, rounds, dev):
    from r2d2_b200 import engine
    c = bench.CONFIGS[name]
    arms = {k: bench.Arm(engine, dict(c, **v), dev, 0, episodes, data_parallel=False) for k, v in ARMS.items()}
    ms = {k: [] for k in arms}
    for _ in range(rounds):
        for k, arm in arms.items():
            ms[k].append(arm.time_resident(steps, 5, torch.cuda.synchronize))
    launches = {k: arm.launches_per_step for k, arm in arms.items()}
    for arm in arms.values():
        arm.close()
    med = {k: statistics.median(v) for k, v in ms.items()}
    return {"workload": bench.workload_string(name, c), "ms_per_step": ms, "median_ms": med,
            "overhead_pct": 100.0 * (med["r2d2"] / med["default"] - 1.0), "gpu_launches_per_step": launches}


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rescale_bench.py needs a CUDA device")
    torch.cuda.set_device(0)
    dev = torch.device("cuda:0")
    np.random.seed(0)
    out = {"arms": ARMS, "card_before": card(),
           "td_cfg3": td_kernels("cfg3", args.reps), "td_cfg2": td_kernels("cfg2", args.reps),
           "cfg3": iterations("cfg3", 256, args.steps, args.rounds, dev),
           "cfg2": iterations("cfg2", 128, args.steps, args.rounds, dev), "card_after": card()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()

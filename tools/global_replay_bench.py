"""Cost of global sampling on one GPU: replay-fed pipelined iterations (LearnerEngine.step with the write-back + draw
hook) of the local and the global mode at W = 1, arms alternated in one process, at BASELINE.json configs[2] and
configs[1].  Prints one JSON line per config with ms per iteration (median of the rounds) and the hook's launches.

W >= 2 across GPUs needs one process per GPU (torchrun); on a one-GPU machine it is reported as not measured.  Report the
card, power limit and clocks next to the numbers (nvidia-smi --query-gpu=name,power.limit,clocks.sm,clocks.max.sm)."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "pytorch-r2d2-dpg_b200"), os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from learner_harness import episode  # noqa: E402
from r2d2_b200 import engine as E  # noqa: E402
from r2d2_b200 import native as nv  # noqa: E402

CONFIGS = {"cfg2": dict(obs=17, act=6, hidden=256, batch=256, burn_in=40, learning=80, n_step=5),
           "cfg1": dict(obs=24, act=6, hidden=128, batch=32, burn_in=20, learning=40, n_step=5)}


def arm(kw, global_sampling):
    cfg = E.PathConfig(**kw, priority_exponent=0.9, is_exponent=0.6, global_sampling=global_sampling)
    rng = np.random.default_rng(1)
    rp = E.DeviceReplay(cfg, capacity_rows=64 * (cfg.rows + 200))
    rp.add_episodes([episode(rng, cfg, cfg.rows + 150) for _ in range(64)])
    eng = E.LearnerEngine(cfg, seed=1)
    if global_sampling:
        rp.attach_group(eng)
    gen = torch.Generator(device="cuda").manual_seed(2)
    launches = []

    def hook(e, used):
        n0 = nv.lib().r2d2_launch_count()
        rp.update_priorities(used.leaf_idx, used.priority)
        rp.sample_into(e, generator=gen)
        launches.append(nv.lib().r2d2_launch_count() - n0)

    rp.sample_into(eng, generator=gen)
    return eng, rp, hook, launches


def main(steps=30, rounds=5):
    n_gpus = torch.cuda.device_count()
    for name, kw in CONFIGS.items():
        arms = {"local": arm(kw, False), "global": arm(kw, True)}
        ms = {k: [] for k in arms}
        for _ in range(rounds):
            for k, (eng, _, hook, _) in arms.items():          # alternated: local, global, local, ...
                for _ in range(3):
                    eng.step(prefetch=hook)
                torch.cuda.synchronize()
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record()
                for _ in range(steps):
                    eng.step(prefetch=hook)
                t1.record()
                torch.cuda.synchronize()
                ms[k].append(t0.elapsed_time(t1) / steps)
        out = {"config": name, "workload": kw, "W": 1, "gpu": torch.cuda.get_device_name(0),
               "ms_per_iteration": {k: float(np.median(v)) for k, v in ms.items()},
               "rounds": {k: [round(x, 4) for x in v] for k, v in ms.items()},
               "hook_launches": {k: sorted(set(a[3])) for k, a in arms.items()},
               "global_status": arms["global"][1].global_status(),
               "W>=2 across GPUs": "not measured (%d GPU on this machine)" % n_gpus if n_gpus < 2 else
                                   "run one process per GPU under torchrun"}
        print(json.dumps(out), flush=True)
        for eng, rp, _, _ in arms.values():
            rp.close()
            eng.close()


if __name__ == "__main__":
    main()

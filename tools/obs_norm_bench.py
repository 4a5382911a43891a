"""Observation normalisation (PathConfig.obs_norm), off against on, in one process on one GPU.

The two arms alternate over the rounds.  Reported per arm:
  - the gather kernel per draw (r2d2_replay_gather at the drawn leaves into the engine's batch), CUDA events, for the
    device and the host state tier, at cfg-3 (obs 376, act 17, H 512, batch 512) and cfg-2 (obs 17, act 6, H 256,
    batch 256), window 40 + 80 + 5;
  - the replay-fed pipelined learner iteration (step + write-back + next draw in the prefetch hook), CUDA events;
  - r2d2_policy_step (off) and r2d2_policy_step_ex (on) at cfg-3's shape for N = 1, 64, 256 lanes, CUDA events;
  - add_episodes of one cfg-3 actor file (16 episodes of 250 + 5 rows) without and with the observation moments, host
    clock around the call (it synchronises), median of 9.
The card's name, power limit and SM clocks are read in the same process.  Prints one JSON line; --out writes it too.

    python tools/obs_norm_bench.py [--rounds 3] [--steps 10] [--out bench_out/obs_norm.json]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "pytorch-r2d2-dpg_b200"), os.path.join(ROOT, "tools")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from r2d2_b200 import engine  # noqa: E402
from r2d2_b200 import native as nv  # noqa: E402
from r2d2_b200.obs_norm import ObsNormStats  # noqa: E402
from r2d2_b200.policy_step import policy_step  # noqa: E402
from replay_storage_bench import CONFIGS, actor_file, card, events_ms  # noqa: E402

ARMS = ("off", "on")
TIERS = ("device", "host")


class Setup:
    """One shard of 4 actor files and one engine for a config, a state tier and an arm."""

    def __init__(self, name, tier, arm, files):
        self.cfg = engine.PathConfig(**CONFIGS[name], replay_state_memory=tier, obs_norm=arm == "on")
        rows = sum(e[0].shape[0] for f in files for e in f)
        self.rp = engine.DeviceReplay(self.cfg, capacity_rows=rows)
        self.eng = engine.LearnerEngine(self.cfg, seed=1)
        stats = self.eng.obs_norm
        if stats is not None:
            self.rp.attach_obs_norm(stats)
        for f in files:
            self.rp.add_episodes(f, obs_norm=stats)
        if stats is not None:
            stats.exchange()
        self.gen = torch.Generator(device="cuda").manual_seed(0)
        self.rp.sample_into(self.eng, generator=self.gen)
        torch.cuda.synchronize()

    def gather(self):
        e = self.eng
        nv.check(self.rp.lib.r2d2_replay_gather(self.rp._h, nv.dptr(e.leaf_idx, torch.int64), self.cfg.batch,
                                                nv.dptr(e.obs), nv.dptr(e.act), nv.dptr(e.rew), nv.dptr(e.term),
                                                nv.dptr(e.states), nv.current_stream()))

    def step(self):
        def hook(e, used):
            self.rp.update_priorities(used.leaf_idx, used.priority)
            self.rp.sample_into(e, generator=self.gen)
        self.eng.step(prefetch=hook)

    def close(self):
        self.eng.close()
        self.rp.close()


def policy_arms(N):
    c = CONFIGS["cfg3"]
    O, A, H = c["obs"], c["act"], c["hidden"]
    lib = nv.lib()
    g = torch.Generator(device="cuda").manual_seed(N)
    params = [0.05 * torch.randn(lib.r2d2_net_param_count(nv.byref(nv.NetShape(O, A, H, int(k >= 2)))), device="cuda",
                                 generator=g) for k in range(4)]
    obs = 5 * torch.randn(N, O, device="cuda", generator=g)
    s_in = 0.1 * torch.randn(4, 2, N, H, device="cuda", generator=g)
    s_out, mu = torch.empty_like(s_in), torch.empty(N, A, device="cuda")
    ws = torch.empty(lib.r2d2_policy_workspace_floats(nv.byref(nv.NetShape(O, A, H, 0)), N), device="cuda")
    norm = (torch.randn(O, device="cuda", generator=g), torch.rand(O, device="cuda", generator=g) + 0.1, 5.0)
    return {"off": lambda: policy_step(params, obs, s_in, s_out, mu, ws),
            "on": lambda: policy_step(params, obs, s_in, s_out, mu, ws, obs_norm=norm)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("obs_norm_bench needs a CUDA device")
    rng = np.random.default_rng(0)
    out = {"card": card(), "rounds": args.rounds, "steps": args.steps}
    res = {}
    for name in CONFIGS:
        files = [actor_file(engine.PathConfig(**CONFIGS[name]), rng) for _ in range(4)]
        for tier in TIERS:
            for rnd in range(args.rounds):
                for arm in (ARMS if rnd % 2 == 0 else ARMS[::-1]):
                    s = Setup(name, tier, arm, files)
                    for _ in range(3):
                        s.gather()
                    r = res.setdefault(f"{name}/{tier}/{arm}", {"gather_us": [], "iteration_ms": []})
                    r["gather_us"].append(1e3 * events_ms(s.gather, 200))
                    if tier == "device":
                        for _ in range(3):
                            s.step()
                        r["iteration_ms"].append(events_ms(s.step, args.steps))
                    s.close()
    for N in (1, 64, 256):
        fns = policy_arms(N)
        for rnd in range(args.rounds):
            for arm in (ARMS if rnd % 2 == 0 else ARMS[::-1]):
                for _ in range(5):
                    fns[arm]()
                res.setdefault(f"policy_step/N{N}/{arm}", {"us": []})["us"].append(1e3 * events_ms(fns[arm], 500))
    c3 = engine.PathConfig(**CONFIGS["cfg3"])
    f = actor_file(c3, rng)
    rows = sum(e[0].shape[0] for e in f)
    stats = ObsNormStats(c3.obs, 5.0, "cuda")
    for rnd in range(args.rounds):
        for arm in (ARMS if rnd % 2 == 0 else ARMS[::-1]):
            rp = engine.DeviceReplay(c3, capacity_rows=8 * rows)
            kw = {"obs_norm": stats} if arm == "on" else {}
            rp.add_episodes(f, **kw)                              # warm: scratch allocated, modules loaded
            ts = []
            for _ in range(9):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                rp.add_episodes(f, **kw)                          # synchronises before it returns
                ts.append(1e3 * (time.perf_counter() - t0))
            res.setdefault(f"add_episodes/cfg3/{arm}", {"ms": []})["ms"].append(float(np.median(ts)))
            rp.close()
    for r in res.values():
        for m in [m for m in r if isinstance(r[m], list)]:
            v = r[m]
            r[m] = None if not v else {"median": round(float(np.median(v)), 3), "min": round(float(min(v)), 3),
                                       "max": round(float(max(v)), 3)}
    out["results"] = res
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()

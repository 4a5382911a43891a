"""What in-step exploration noise costs on one GPU, in one command:

  1. per-step time from CUDA events over --steps steps after --warmup, at the cfg-1, cfg-2 and cfg-3 shapes and
     N in {1, 16, 64, 256}: r2d2_policy_step alone; r2d2_policy_step followed by a stream synchronisation (what
     PolicyStepper does every step); r2d2_policy_step_explore in gaussian and in ou mode, whose sigma check reads sigma
     back and synchronises the stream inside the call;
  2. ActorPool env-steps/s with the synthetic env, R2D2_EXPLORATION=reference against gaussian, alternated twice.

    python tools/exploration_bench.py [--steps 1000] [--warmup 100] [--pool-steps 300] [--out result.json]

Nothing is written into the tree: the pools run in a temporary directory.
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from actor_pool_bench import CFGS, LANES, NETS, card, event_time, model_dict  # noqa: E402

POOL_CFG, POOL_LANES = "cfg-2", (16, 256)


def bench_kernels(steps, warmup):
    from r2d2_b200 import native as nv
    from r2d2_b200.actor_priority import _flat
    from r2d2_b200.exploration import Exploration
    from r2d2_b200.policy_step import policy_step
    lib = nv.lib()
    rows = []
    for cfg, (O, A, H) in CFGS.items():
        md = model_dict(O, A, H)
        params = [_flat(md[n], "cuda") for n in NETS]
        for N in LANES:
            g = torch.Generator(device="cuda").manual_seed(N)
            obs = torch.randn((N, O), device="cuda", generator=g)
            s_in = 0.1 * torch.randn((4, 2, N, H), device="cuda", generator=g)
            s_out = torch.empty_like(s_in)
            mu, act = torch.empty((N, A), device="cuda"), torch.empty((N, A), device="cuda")
            ws = torch.empty(lib.r2d2_policy_workspace_floats(nv.byref(nv.NetShape(O, A, H, 0)), N), device="cuda")
            stream = torch.cuda.current_stream()
            r = {"cfg": cfg, "O": O, "A": A, "H": H, "N": N}
            r["policy_step_us"] = event_time(lambda: policy_step(params, obs, s_in, s_out, mu, ws), steps, warmup)

            def synced():
                policy_step(params, obs, s_in, s_out, mu, ws)
                stream.synchronize()
            r["policy_step_sync_us"] = event_time(synced, steps, warmup)
            opt = Exploration("ou", 0.4, 0.05, 256, seed=1)
            sigma = torch.from_numpy(opt.sigmas(range(N))).cuda()
            ids = torch.arange(N, dtype=torch.int32, device="cuda")
            ou = torch.zeros((N, A), device="cuda")
            for mode in ("gaussian", "ou"):
                ex = dict(mode=mode, seed=1, step=0, one_minus_theta=float(opt.one_minus_theta), actor_id=ids,
                          sigma=sigma, ou_state=ou if mode == "ou" else None)
                r[mode + "_us"] = event_time(lambda: policy_step(params, obs, s_in, s_out, mu, ws, exploration=ex,
                                                                 action=act), steps, warmup)
            for k in ("policy_step_us", "policy_step_sync_us", "gaussian_us", "ou_us"):
                r[k] = round(r[k], 2)
            rows.append(r)
            print("%-5s N=%3d  policy_step %7.2f us | + sync %7.2f us | explore gaussian %7.2f us | ou %7.2f us"
                  % (cfg, N, r["policy_step_us"], r["policy_step_sync_us"], r["gaussian_us"], r["ou_us"]), flush=True)
    return rows


def bench_pool(mode, n_lanes, steps):
    O, A, H = CFGS[POOL_CFG]
    env = {"R2D2_OBS_SIZE": str(O), "R2D2_N_ACTIONS": str(A), "R2D2_HIDDEN": str(H)}
    if mode != "reference":
        env.update({"R2D2_EXPLORATION": mode, "R2D2_EXPLORATION_SIGMA": "0.4", "R2D2_EXPLORATION_SIGMA_MIN": "0.05",
                    "R2D2_EXPLORATION_ACTORS": str(n_lanes)})
    saved = {k: os.environ.get(k) for k in list(env) + ["R2D2_EXPLORATION"]}
    os.environ.update(env)
    from actor_pool import ActorPool
    with tempfile.TemporaryDirectory() as d:
        cwd = os.getcwd()
        os.chdir(d)
        try:
            os.makedirs("memory_data")
            os.makedirs("model_data")
            pool = ActorPool(range(n_lanes), device="cuda")
            for e in pool.envs:
                e.episode_len = 100                         # episode ends (priorities, files) inside the window
            pool.run(max_steps=20)
            pool.host_time = pool.device_time = 0.0
            t0 = time.perf_counter()
            pool.run(max_steps=steps)
            wall = time.perf_counter() - t0
        finally:
            os.chdir(cwd)
            for k, v in saved.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
    r = {"mode": mode, "cfg": POOL_CFG, "lanes": n_lanes, "pool_steps": steps,
         "env_steps_per_s": round(n_lanes * steps / wall, 1), "host_env_s": round(pool.host_time, 3),
         "device_step_s": round(pool.device_time, 3), "wall_s": round(wall, 3)}
    print("pool %-9s %s lanes=%3d: %8.0f env-steps/s (host env %.2f s, device step %.2f s, wall %.2f s)"
          % (mode, POOL_CFG, n_lanes, r["env_steps_per_s"], r["host_env_s"], r["device_step_s"], wall), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=100)
    ap.add_argument("--pool-steps", type=int, default=300)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("exploration_bench needs a GPU")
    info = card()
    print(info, flush=True)
    kernels = bench_kernels(args.steps, args.warmup)
    pools = [bench_pool(mode, n, args.pool_steps) for n in POOL_LANES for _ in range(2)
             for mode in ("reference", "gaussian")]
    out = {"card": info, "kernels": kernels, "pool": pools, "card_after": card()}
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)
    ratios = [p["env_steps_per_s"] for p in pools]
    print("pool gaussian / reference env-steps/s:",
          [round(ratios[i + 1] / ratios[i], 3) for i in range(0, len(ratios), 2)], flush=True)
    print(json.dumps({"kernels": len(kernels), "pools": len(pools), "mean_pool_ratio":
                      float(np.mean([ratios[i + 1] / ratios[i] for i in range(0, len(ratios), 2)]))}))


if __name__ == "__main__":
    main()

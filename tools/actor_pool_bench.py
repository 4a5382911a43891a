"""Actor-side step measurements on one GPU, in one command:

  1. r2d2_policy_step kernel time alone (CUDA events over --steps steps after --warmup) at the cfg-1, cfg-2 and cfg-3
     shapes and N in {1, 16, 64, 256}, with bytes and FLOPs computed from the shapes and the share of the larger of
     the two data-sheet bounds (H100 SXM: 3.35 TB/s HBM3, 67 TFLOP/s FP32);
  2. the same step done the two ways available before it, at the same N: four r2d2_lstm_net_forward(T = 1) calls, and
     the models.py nets in torch eager on the GPU;
  3. ActorPool env-steps/s end to end with the synthetic env, split into host env time and device time;
  4. the drop-in CPU Actor's env-steps/s on one core (the reference's cost per host core).

    python tools/actor_pool_bench.py [--steps 1000] [--warmup 100] [--out result.json]

Nothing is written into the tree: the pool and the CPU actor run in a temporary directory.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "pytorch-r2d2-dpg_b200")
for _p in (ROOT, PKG):
    if _p not in sys.path:
        sys.path.insert(0, _p)

CFGS = {"cfg-1": (3, 1, 128), "cfg-2": (17, 6, 256), "cfg-3": (376, 17, 512)}   # (obs, act, hidden), BASELINE.json
LANES = (1, 16, 64, 256)
HBM_BPS, FP32_FLOPS = 3.35e12, 67e12
NETS = ("actor", "target_actor", "critic", "target_critic")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": q[torch.cuda.current_device()] if q else "unavailable"}


def work(O, A, H, N):
    """(bytes, flops) of one step: every weight the step uses read once (the critics' heads are not), obs / mu / states
    moved once."""
    macs_actor = H * O + 8 * H * H + A * H
    macs_critic = H * (O + A) + 8 * H * H
    n_params = 2 * (macs_actor + H + 8 * H + A) + 2 * (macs_critic + H + 8 * H)
    bytes_ = 4 * (n_params + N * (O + A) + 2 * 4 * 2 * N * H)
    return bytes_, 2 * N * 2 * (macs_actor + macs_critic)


def event_time(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / steps                     # us per step


def model_dict(O, A, H):
    from actor_pool import initial_model_dict
    torch.manual_seed(0)
    md = initial_model_dict(O, A, H)
    for sd in md.values():
        sd["l3.weight"].uniform_(-0.1, 0.1)
    return md


def bench_kernels(steps, warmup):
    from actor_pool import ModelsStepper
    from r2d2_b200 import native as nv
    from r2d2_b200.actor_priority import _flat
    from r2d2_b200.policy_step import policy_step
    lib = nv.lib()
    rows = []
    for cfg, (O, A, H) in CFGS.items():
        md = model_dict(O, A, H)
        params = [_flat(md[n], "cuda") for n in NETS]
        eager = ModelsStepper(O, A, H, 1, device="cuda", max_episode_steps=1)
        eager.load(md)
        for N in LANES:
            g = torch.Generator(device="cuda").manual_seed(N)
            obs = torch.randn((N, O), device="cuda", generator=g)
            s_in = 0.1 * torch.randn((4, 2, N, H), device="cuda", generator=g)
            s_out = torch.empty_like(s_in)
            mu = torch.empty((N, A), device="cuda")
            ws = torch.empty(lib.r2d2_policy_workspace_floats(nv.byref(nv.NetShape(O, A, H, 0)), N), device="cuda")
            t_step = event_time(lambda: policy_step(params, obs, s_in, s_out, mu, ws), steps, warmup)

            # before: four r2d2_lstm_net_forward(T = 1) chains, one per net
            sh_a, sh_c = nv.NetShape(O, A, H, 0), nv.NetShape(O, A, H, 1)
            wsz = max(lib.r2d2_net_workspace_floats(nv.byref(s), 1, N, 1) for s in (sh_a, sh_c))
            wss = [torch.empty(wsz, device="cuda") for _ in range(4)]
            mu_t = torch.empty_like(mu)
            q = torch.empty_like(mu)
            st = nv.current_stream()

            def chains():
                for k, (sh, act, out) in enumerate(((sh_a, None, mu), (sh_a, None, mu_t), (sh_c, mu, q),
                                                    (sh_c, mu_t, q))):
                    nv.check(lib.r2d2_lstm_net_forward(nv.byref(sh), nv.dptr(params[k]), nv.dptr(obs), nv.dptr(act),
                                                       nv.dptr(s_in[k, 0]), nv.dptr(s_in[k, 1]), 1, N, 1, 0,
                                                       nv.dptr(out), nv.dptr(wss[k]), st))
            t_chain = event_time(chains, max(100, steps // 5), warmup)

            # before: torch eager models.py nets on the GPU
            a_net, ta_net, c_net, tc_net = eager.nets

            @torch.no_grad()
            def eager_step():
                for k, net in enumerate(eager.nets):
                    net.set_state(s_in[k, 0], s_in[k, 1])
                m = a_net(obs)
                c_net(obs, m)
                tc_net(obs, ta_net(obs))
            t_eager = event_time(eager_step, max(100, steps // 5), warmup)

            b, f = work(O, A, H, N)
            t_bytes, t_flops = b / HBM_BPS * 1e6, f / FP32_FLOPS * 1e6
            bound = "bytes" if t_bytes >= t_flops else "fp32"
            rows.append({"cfg": cfg, "O": O, "A": A, "H": H, "N": N, "policy_step_us": round(t_step, 2),
                         "four_chains_us": round(t_chain, 2), "torch_eager_us": round(t_eager, 2),
                         "MB": round(b / 1e6, 2), "MFLOP": round(f / 1e6, 1), "bound": bound,
                         "bound_us": round(max(t_bytes, t_flops), 2),
                         "share_of_bound": round(max(t_bytes, t_flops) / t_step, 3)})
            print("%-5s N=%3d  policy_step %8.2f us | 4 chains %8.1f us | eager %8.1f us | %7.2f MB %8.1f MFLOP | "
                  "%s bound %6.2f us -> %5.1f %%" % (cfg, N, t_step, t_chain, t_eager, b / 1e6, f / 1e6, bound,
                                                   max(t_bytes, t_flops), 100 * max(t_bytes, t_flops) / t_step),
                  flush=True)
    return rows


def bench_pool(cfg, n_lanes, steps):
    O, A, H = CFGS[cfg]
    os.environ.update({"R2D2_OBS_SIZE": str(O), "R2D2_N_ACTIONS": str(A), "R2D2_HIDDEN": str(H)})
    from actor_pool import ActorPool
    with tempfile.TemporaryDirectory() as d:
        cwd = os.getcwd()
        os.chdir(d)
        try:
            os.makedirs("memory_data")
            os.makedirs("model_data")
            pool = ActorPool(range(n_lanes), device="cuda")
            for env in pool.envs:
                env.episode_len = 100                       # episode ends (priorities, files) inside the window
            pool.run(max_steps=20)
            pool.host_time = pool.device_time = 0.0
            t0 = time.perf_counter()
            pool.run(max_steps=steps)
            wall = time.perf_counter() - t0
        finally:
            os.chdir(cwd)
    r = {"cfg": cfg, "lanes": n_lanes, "pool_steps": steps, "env_steps_per_s": round(n_lanes * steps / wall, 1),
         "host_env_s": round(pool.host_time, 3), "device_step_s": round(pool.device_time, 3),
         "episode_end_s": round(wall - pool.host_time - pool.device_time, 3), "wall_s": round(wall, 3)}
    print("pool %s lanes=%d: %.0f env-steps/s (host env %.2f s, device step %.2f s, episode ends %.2f s, wall %.2f s)"
          % (cfg, n_lanes, r["env_steps_per_s"], r["host_env_s"], r["device_step_s"], r["episode_end_s"], wall),
          flush=True)
    return r


def bench_cpu_actor(cfg, steps):
    O, A, H = CFGS[cfg]
    os.environ.update({"R2D2_OBS_SIZE": str(O), "R2D2_N_ACTIONS": str(A), "R2D2_HIDDEN": str(H),
                       "R2D2_ACTOR_DEVICE": "cpu"})
    import actor
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    with tempfile.TemporaryDirectory() as d:
        cwd = os.getcwd()
        os.chdir(d)
        try:
            a = actor.Actor(0)
            a.env.episode_len = steps
            a.calc_priorities = lambda: None                   # per-step cost only: the episode-end pass is not timed
            t0 = time.perf_counter()
            a.run(max_episodes=1)
            wall = time.perf_counter() - t0
        finally:
            os.chdir(cwd)
            torch.set_num_threads(threads)
    r = {"cfg": cfg, "steps": steps, "env_steps_per_s_one_core": round(steps / wall, 1)}
    print("drop-in CPU Actor %s, 1 thread: %.1f env-steps/s" % (cfg, r["env_steps_per_s_one_core"]), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=100)
    ap.add_argument("--pool-steps", type=int, default=300)
    ap.add_argument("--cpu-steps", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("actor_pool_bench.py measures on a GPU; none is visible")
    torch.cuda.set_device(0)
    info = card()
    print("device:", info["device"], "| nvidia-smi name, power.limit, clocks.sm, clocks.max.sm:", info["nvidia_smi"],
          flush=True)
    res = {"card": info, "kernels": bench_kernels(args.steps, args.warmup),
           "pool": [bench_pool("cfg-3", n, args.pool_steps) for n in (16, 64)] + [bench_pool("cfg-2", 64, args.pool_steps)],
           "cpu_actor": [bench_cpu_actor(c, args.cpu_steps) for c in ("cfg-3", "cfg-2")]}
    res["card_after"] = card()["nvidia_smi"]
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

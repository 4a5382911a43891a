"""Where a data-parallel iteration spends its time (dev tool): CUDA events at the phase boundaries of LearnerEngine.step,
averaged per rank.  torchrun --nproc-per-node N tools/dp_phase_time.py [variant ...]
variants: peer | peer_seq (next batch drawn at the end of the step: no target chains ahead).  One process without
torchrun times the single-GPU step."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "pytorch-r2d2-dpg_b200"))
import torch  # noqa: E402

import bench  # noqa: E402
from r2d2_b200 import engine, native as nv  # noqa: E402
from r2d2_b200.dist_env import DistEnv  # noqa: E402

env = DistEnv.from_environ()
torch.cuda.set_device(env.local_rank)
dev = torch.device(f"cuda:{env.local_rank}")
dist = env.init_process_group("nccl", device=dev)
STEPS, WARM = 40, 6
NAMES = ["critic_phase", "flush(prev actor step)", "tree update + sample", "target_phase(next)", "actor_forward", "actor_phase", "finish / late sample"]


def run(variant):
    if variant not in ("peer", "peer_seq"):
        raise SystemExit(f"unknown variant {variant!r}: peer | peer_seq")
    os.environ["R2D2_DP_MODE"] = "peer"
    arm = bench.Arm(engine, bench.CONFIGS["cfg3"], dev, env.rank, 96, data_parallel=dist is not None)
    eng, lib = arm.eng, arm.eng.lib
    mode = eng._dp_mode if dist is not None else "single"
    if mode == "defer":
        raise SystemExit("no peer-mapped gradient buffer: the exchange fell back to NCCL, which this tool does not spell out")
    pipelined = variant == "peer"
    arm.rp.sample_into(eng, generator=arm.gen)
    scale = 1.0 / eng.world
    evs = [[torch.cuda.Event(enable_timing=True) for _ in range(len(NAMES) + 1)] for _ in range(STEPS)]

    def one(ev):
        """LearnerEngine.step(prefetch=...) for mode peer / one GPU spelled out, with events between the calls"""
        s = nv.current_stream()
        rec = (lambda i: ev[i].record()) if ev is not None else (lambda i: None)
        rec(0)
        if eng._fill_slot != eng._lib_slot:
            nv.check(lib.r2d2_learner_select_batch(eng._h, eng._fill_slot))
            eng._lib_slot = eng._fill_slot
        eng._targets_ahead = False
        if eng._pending_finish and eng._finish_updates_targets():
            eng.flush()
        nv.check(lib.r2d2_learner_critic_phase(eng._h, s)); rec(1)
        eng.flush()
        rec(2)
        ahead = pipelined and not eng._finish_updates_targets()
        if ahead:
            eng._run_prefetch(arm._next_batch)
            rec(3)
            nv.check(lib.r2d2_learner_target_phase(eng._h, eng._fill_slot, s))
        else:
            rec(3)
        rec(4)
        nv.check(lib.r2d2_learner_actor_forward(eng._h, s)); rec(5)
        nv.check(lib.r2d2_learner_actor_phase(eng._h, scale, s)); rec(6)
        if mode == "peer":
            eng._pending_finish = True
        else:
            nv.check(lib.r2d2_learner_finish_phase(eng._h, scale, s))
        if not ahead:
            eng._run_prefetch(arm._next_batch)
        rec(7)

    for _ in range(WARM):
        one(None)
    torch.cuda.synchronize()
    if dist is not None:
        dist.barrier()
    import ctypes
    cnt = (ctypes.c_ulonglong * 6)()
    if eng._peer_buf is not None:
        nv.check(lib.r2d2_learner_peer_counters(eng._h, cnt, 1, nv.current_stream()))
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for i in range(STEPS):
        one(evs[i])
    t1.record()
    torch.cuda.synchronize()
    seg = [sum(e[i].elapsed_time(e[i + 1]) for e in evs) / STEPS for i in range(len(NAMES))]
    total = t0.elapsed_time(t1) / STEPS
    extra = [0.0] * 6
    if eng._peer_buf is not None:
        nv.check(lib.r2d2_learner_peer_counters(eng._h, cnt, 0, nv.current_stream()))
        extra = [cnt[i] * 1e-6 / STEPS for i in range(6)]
    row = torch.tensor(seg + [total] + extra, device=dev)
    rows = [torch.zeros_like(row) for _ in range(env.world)]
    if dist is not None:
        dist.all_gather(rows, row)
    else:
        rows = [row]
    if env.rank == 0:
        print(f"== {variant} (mode {mode}) ms per iteration, one column per rank")
        for i, n in enumerate(NAMES + ["TOTAL", "slice sum (critic): waiting", "slice sum (actor): waiting",
                               "slice sum (critic): total", "slice sum (actor): total", "wait kernel (critic)",
                               "wait kernel (actor)"]):
            print(f"  {n:26s} " + " ".join(f"{r[i].item():8.3f}" for r in rows))
        sys.stdout.flush()
    arm.close()
    if dist is not None:
        dist.barrier()


for v in (sys.argv[1:] or ["peer", "peer_seq"]):
    run(v)
if dist is not None:
    dist.destroy_process_group()

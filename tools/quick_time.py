"""Rough device timing of one learner iteration (dev tool; bench.py is the contract)."""
import json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "pytorch-r2d2-dpg_b200")]
import numpy as np, torch
from r2d2_b200 import engine, native as nv
from oracle import ref_port

def run(obs, act, hidden, batch, burn_in, learning, iters=10):
    cfg = engine.PathConfig(obs=obs, act=act, hidden=hidden, batch=batch, burn_in=burn_in, learning=learning)
    eng = engine.LearnerEngine(cfg)
    pc = ref_port.PathConfig(obs=obs, act=act, hidden=hidden, batch=batch, burn_in=burn_in, learning=learning)
    eng.set_batch(ref_port.synthetic_batch(pc, 0))
    for _ in range(3): eng.step()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    tot = np.zeros(3)
    s = nv.current_stream()
    for _ in range(iters):
        ev[0].record(); nv.check(eng.lib.r2d2_learner_critic_phase(eng._h, s))
        ev[1].record(); nv.check(eng.lib.r2d2_learner_actor_phase(eng._h, 1.0, s))
        ev[2].record(); nv.check(eng.lib.r2d2_learner_finish_phase(eng._h, 1.0, s))
        ev[3].record(); torch.cuda.synchronize()
        tot += [ev[i].elapsed_time(ev[i+1]) for i in range(3)]
    tot /= iters
    out = {"cfg": [obs, act, hidden, batch, burn_in, learning], "ms_phase": tot.round(4).tolist(), "ms_iter": round(float(tot.sum()), 4),
           "seq_steps_per_s": batch * learning / (tot.sum() * 1e-3), "launches": eng.launches_per_iteration}
    print(json.dumps(out)); return out

CFGS = {"cfg1": (24, 6, 128, 32, 20, 40), "cfg2": (17, 6, 256, 256, 40, 80), "cfg3": (376, 17, 512, 512, 40, 80),
        "cfg3s": (376, 17, 512, 64, 40, 80)}

if __name__ == "__main__":
    names = sys.argv[1:] or ["cfg1", "cfg2"]
    res = [run(*CFGS[n], iters=5 if n.startswith("cfg3") else 10) for n in names]
    os.makedirs(os.path.join(ROOT, "bench_out"), exist_ok=True)
    json.dump(res, open(os.path.join(ROOT, "bench_out", "quick_time_" + "_".join(names) + ".json"), "w"))

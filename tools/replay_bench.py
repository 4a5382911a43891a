"""BASELINE.json configs[3]: GPU-resident prioritized replay shard (2M sequence starts sharded 8-way = 250k starts per GPU):
sum-tree sample + gather + priority-update throughput, and index bit-exactness against the C restatement."""
import json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "pytorch-r2d2-dpg_b200")]
import numpy as np, torch
from r2d2_b200 import engine
from oracle.sumtree import SumTreeOracle

def main():
    cfg = engine.PathConfig(obs=17, act=6, hidden=256, batch=256, burn_in=40, learning=80, n_step=5)
    n_ep, E = 1000, 250 + cfg.burn_in + cfg.learning          # 250 starts per episode -> 250k starts
    n_rows = E + cfg.n_step
    rp = engine.DeviceReplay(cfg, capacity_rows=n_ep * n_rows)
    oracle = SumTreeOracle(n_ep * n_rows)
    rng = np.random.default_rng(0)
    t0 = time.time()
    obs = rng.standard_normal((n_rows, cfg.obs), dtype=np.float32); act = rng.uniform(-1, 1, (n_rows, cfg.act)).astype(np.float32)
    rew = rng.standard_normal(n_rows, dtype=np.float32); term = np.zeros(n_rows, np.float32); term[E:] = 1
    st = (0.1 * rng.standard_normal((E, 4, 2, cfg.hidden), dtype=np.float32))
    for e in range(n_ep):
        p = rng.uniform(0.01, 1.0, 250).astype(np.float32)
        rp.add_episode(obs, act, rew, term, st, p)
        oracle.set_range(e * n_rows, p)
    torch.cuda.synchronize()
    ingest_s = time.time() - t0
    eng = engine.LearnerEngine(cfg)
    gen = torch.Generator(device="cuda").manual_seed(0)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = {"sequence_starts": n_ep * 250, "rows": n_ep * n_rows, "tree_levels": rp.stats()["tree_levels"], "ingest_s": round(ingest_s, 2)}
    # (a) index draw only, big batches
    u = torch.rand(1 << 20, device="cuda", generator=gen)
    for _ in range(3): leaf = rp.sample_indices(u)
    ev0.record()
    for _ in range(10): leaf = rp.sample_indices(u)
    ev1.record(); torch.cuda.synchronize()
    out["draws_per_s"] = 10 * u.numel() / (ev0.elapsed_time(ev1) * 1e-3)
    out["indices_bit_exact_vs_c_tree"] = bool(np.array_equal(leaf.cpu().numpy(), oracle.sample(u.cpu().numpy())))
    # (b) learner-shaped: sample 256 + gather the time-major batch into the engine, then write 256 priorities back
    for _ in range(5): rp.sample_into(eng, generator=gen)
    ev0.record()
    for _ in range(200): rp.sample_into(eng, generator=gen)
    ev1.record(); torch.cuda.synchronize()
    ms = ev0.elapsed_time(ev1) / 200
    batch_bytes = 4 * (cfg.rows * cfg.batch * (cfg.obs + cfg.act + 2) + 8 * cfg.batch * cfg.hidden)
    out["sample_gather_us"] = ms * 1e3
    out["sample_gather_sequences_per_s"] = cfg.batch / (ms * 1e-3)
    out["gather_GBps_read_plus_write"] = 2 * batch_bytes / (ms * 1e-3) / 1e9
    prio = torch.rand(cfg.batch, device="cuda")
    for _ in range(5): rp.update_priorities(eng.leaf_idx, prio)
    ev0.record()
    for _ in range(200): rp.update_priorities(eng.leaf_idx, prio)
    ev1.record(); torch.cuda.synchronize()
    out["update_us_per_256"] = ev0.elapsed_time(ev1) / 200 * 1e3
    out["updates_per_s"] = cfg.batch / (ev0.elapsed_time(ev1) / 200 * 1e-3)
    # bit-exactness after updates
    li = eng.leaf_idx.cpu().numpy(); oracle.update_batch(li, prio.cpu().numpy())
    u2 = torch.rand(100000, device="cuda", generator=gen)
    out["indices_bit_exact_after_update"] = bool(np.array_equal(rp.sample_indices(u2).cpu().numpy(), oracle.sample(u2.cpu().numpy())))
    print(json.dumps(out))
    os.makedirs(os.path.join(ROOT, "bench_out"), exist_ok=True)
    json.dump(out, open(os.path.join(ROOT, "bench_out", "replay_bench.json"), "w"), indent=1)

if __name__ == "__main__":
    main()

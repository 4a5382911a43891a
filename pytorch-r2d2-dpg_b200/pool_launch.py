"""`python pool_launch.py N_ACTORS [N_POOLS]`: the reference's r2d2.py (learner + N_ACTORS actor processes) with the
actors stepped in N_POOLS `actor_pool.ActorPool` processes instead (default 1).  Pool p runs actor ids p, p + N_POOLS,
p + 2 N_POOLS, ..., so ids 0 .. N_ACTORS-1 are covered once and each id writes its own memory{id}.pt: the learner,
including its rank sharding (actor i belongs to rank i mod WORLD_SIZE), is unchanged.  Every pool uses the current CUDA
device; set CUDA_VISIBLE_DEVICES to place it."""
import os
import sys

import torch.multiprocessing as mp

from actor_pool import actor_pool_process
from learner import learner_process


def run(n_actors, n_pools=1):
    os.makedirs('./model_data', exist_ok=True)
    os.makedirs('./memory_data', exist_ok=True)
    ctx = mp.get_context('spawn')
    processes = [ctx.Process(target=learner_process, args=(n_actors,))]
    for p in range(n_pools):
        processes.append(ctx.Process(target=actor_pool_process, args=(list(range(p, n_actors, n_pools)),)))
    for proc in processes:
        proc.start()
    for proc in processes:
        proc.join()


if __name__ == '__main__':
    n_actors = int(sys.argv[1]) if len(sys.argv) > 1 else 16          # r2d2.py:13 n_actors = 16
    n_pools = int(sys.argv[2]) if len(sys.argv) > 2 else 1
    if not 1 <= n_pools <= n_actors:
        sys.exit("N_POOLS must be between 1 and N_ACTORS")
    run(n_actors, n_pools)

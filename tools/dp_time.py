#!/usr/bin/env python
"""tools/dp_time.py -- env-steps/s of the training drivers' iteration (collect + updates + exchange) at 1 rank, or at N ranks under torchrun.

    python tools/dp_time.py --config idqn                          # BASELINE.json configs[1]: IDQN, Foraging-8x8-2p-3f-v3, 4096 envs/GPU, batch 1024
    python tools/dp_time.py --config ippo                          # configs[4]: IPPO, rware-tiny-4ag-v2, 2048 envs/GPU
    torchrun --nproc-per-node 2 tools/dp_time.py --config idqn     # two ranks (weak scaling: the envs per GPU stay)

One iteration is what dqn/train.py and ac/train.py do per loop turn, through the same functions: every rank collects one episode per env, the
env steps are summed over ranks, then the updates run with the exchange the driver would choose (update_n alone on one rank; the in-kernel peer
exchange or the all-reduce between update_grads and update_apply on several).  Prints one JSON line (rank 0) with the card and its power limit.
Two ranks that share one device measure contention, not scaling: the line says so.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

CONFIGS = {
    "idqn": dict(baseline=1, args=["+algorithm=idqn", "env.name=lbforaging:Foraging-8x8-2p-3f-v3", "env.time_limit=25", "env.parallel_envs=4096",
                                   "algorithm.batch_size=1024", "algorithm.buffer_size=65536", "algorithm.training_start=0"]),
    "ippo": dict(baseline=4, args=["+algorithm=ippo", "env.name=rware:rware-tiny-4ag-v2", "env.time_limit=500", "env.parallel_envs=2048"]),
}


def gpu_info(torch, dev):
    info = {"name": torch.cuda.get_device_name(dev), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(dev)], capture_output=True, text=True, timeout=60)
        info["power_limit_w"] = float(out.stdout.strip().splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        pass
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="idqn", choices=sorted(CONFIGS))
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("overrides", nargs="*", help="extra config overrides, e.g. env.parallel_envs=1024")
    a = ap.parse_args()

    import torch

    from codebase_b200 import distributed
    from codebase_b200.config import compose, instantiate
    from codebase_b200.native_env import TrajStore
    from codebase_b200.utils.envs import make_env

    cfg = compose(CONFIGS[a.config]["args"] + ["seed=0"] + a.overrides)
    dp = distributed.init(cfg)
    T, P = int(cfg.env.time_limit), int(cfg.env.parallel_envs)
    env = make_env(0, name=cfg.env.name, time_limit=T, parallel_envs=P, env_gid0=distributed.shard(dp.rank, P), wrappers=cfg.env.wrappers)
    algo = cfg.algorithm
    dqn = algo._target_.startswith("dqn.")
    torch.manual_seed(0)
    if dqn:
        from codebase_b200.dqn import train as drv

        model = instantiate(algo.model, env.single_observation_space, env.single_action_space, algo, max_batch=algo.batch_size, max_episode_length=T)
        dp.sync_learner(model)
        peer = drv.attach_peer_exchange(model, dp)
        rb = TrajStore(int(algo.buffer_size), env.n_agents, T, env.cfg.obs_dim, env.native.device)
        coll = drv.Collector(env, model, T)
        U, B, seed = P, int(algo.batch_size), 7919 * dp.rank
        exchange = "none" if not dp.active else ("in-kernel peer exchange" if peer else f"{dp.backend} all-reduce between update_grads and update_apply")
    else:
        from codebase_b200.ac import train as drv

        model = instantiate(algo.model, env.single_observation_space, env.single_action_space, algo, max_envs=P, max_episode_length=T)
        dp.sync_learner(model)
        coll = drv.Collector(env, model, T, algo.use_proper_termination)
        exchange = "none" if not dp.active else f"{dp.backend} all-reduce between the gradient and apply calls"
    state = dict(pos=0, updates=0, step=0)

    def iteration():
        if dqn:
            final_len, _ = coll.collect(rb, state["pos"] % rb.capacity, 0.5)
            n = drv.iteration_env_steps(final_len, dp)
            state["pos"] += P
            n_valid = min(state["pos"], rb.capacity)
            if dp.active and not peer:
                model.update_n_allreduce(rb, B, n_valid, seed, state["updates"], U, dp.all_reduce_)
            else:
                model.update_n(rb, B, n_valid, seed, state["updates"], U)
            state["updates"] += U
        else:
            final_len, _ = coll.collect()
            if dp.active:
                model.update_allreduce(coll.batch, P, state["step"], dp.all_reduce_)
            else:
                model.update_from_store(coll.batch, P, state["step"])
            n = drv.iteration_env_steps(int(final_len.max().item()), P, dp)
        state["step"] += n
        return n

    for _ in range(a.warmup):
        iteration()
    torch.cuda.synchronize()
    dp.gather_objects(None)
    t0 = time.perf_counter()
    steps = sum(iteration() for _ in range(a.iters))
    torch.cuda.synchronize()
    secs = max(dp.gather_objects(time.perf_counter() - t0))
    shared = dp.active and not dp.own_device
    if dp.is_main:
        print(json.dumps({"config": a.config, "baseline_config": CONFIGS[a.config]["baseline"], "ranks": dp.world, "envs_per_rank": P,
                          "exchange": exchange, "env_steps_per_s": steps / secs, "ms_per_iteration": 1e3 * secs / a.iters, "iterations": a.iters,
                          "ranks_share_a_device": shared, "gpu": gpu_info(torch, torch.cuda.current_device()),
                          "note": "ranks share one device: contention, not scaling" if shared else None}))
    distributed.finish()


if __name__ == "__main__":
    main()

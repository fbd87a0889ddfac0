"""Timings of the Level-Based Foraging grid observation (DESIGN.md §4.1, §7b):

    python tools/lbf_grid_time.py [--out DIR]

prints the GPU's name and power limit, then
  * the env-step kernel (autoreset, explicit actions) per launch at 4 096 and 65 536 envs for 8x8-2p-3f with the vector observation, grid-2s
    and grid-1s: CUDA events over 200 launches, with the achieved HBM bytes/s from the algorithmic byte count below;
  * one IA2C training iteration on Foraging-grid-2s-8x8-2p-3f-v3 at 4 096 envs (T = 25): collection and update apart.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.rware_time import HBM_PEAK, gpu_info  # noqa: E402

IDS = {"vector": "lbforaging:Foraging-8x8-2p-3f-v3", "grid-2s": "lbforaging:Foraging-grid-2s-8x8-2p-3f-v3",
       "grid-1s": "lbforaging:Foraging-grid-1s-8x8-2p-3f-v3"}


def step_bytes(cfg) -> int:
    """Algorithmic HBM bytes of one env-step: 2 * S_state + N * (4 + 4 D + 4) + 2.  S_state: field at its 16-byte pitch, one player word,
    one float episode return per agent, step / food_spawned / ep_len / episode_idx, the active flag.  Per agent: the action read, the
    observation and the reward written; then the done and truncated flags."""
    N, D, pitch = cfg.n_agents, cfg.obs_dim, (cfg.rows * cfg.cols + 15) // 16 * 16
    state = pitch + 4 * N + 4 * N + 4 * 4 + 1
    return 2 * state + N * (4 + 4 * D + 4) + 2


def time_env_step(kind: str, E: int, launches: int = 200) -> dict:
    from codebase_b200.lbf import NativeLbf, parse_env_id

    cfg = parse_env_id(IDS[kind], 25)
    env = NativeLbf(cfg, E, seed=1)
    env.reset()
    acts = torch.randint(0, 6, (E, cfg.n_agents), dtype=torch.int32, device="cuda")
    for _ in range(20):
        env.step(acts, autoreset=True)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(launches):
        env.step(acts, autoreset=True)
    b.record()
    torch.cuda.synchronize()
    us = a.elapsed_time(b) * 1e3 / launches
    by = step_bytes(cfg) * E
    env.close()
    return dict(kind=kind, D=cfg.obs_dim, envs=E, us_per_launch=us, env_steps_per_s=E / us * 1e6, bytes_per_env_step=step_bytes(cfg),
                hbm_bytes_per_s=by / us * 1e6, share_of_3_35_TBps=by / us * 1e6 / HBM_PEAK)


def time_ia2c(P: int = 4096, T: int = 25, iters: int = 5) -> dict:
    from codebase_b200.ac.model import A2CNetwork
    from codebase_b200.ac.train import Collector
    from codebase_b200.utils.envs import make_env

    envs = make_env(0, name=IDS["grid-2s"], time_limit=T, parallel_envs=P, wrappers=["FlattenObservation"])
    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=0.5, n_steps=5, entropy_coef=0.01, value_loss_coef=0.5,
                                target_update_interval_or_tau=200, standardise_returns=False)
    net = types.SimpleNamespace(layers=[128, 128], parameter_sharing=False, use_rnn=False, use_orthogonal_init=True, centralised=False)
    m = A2CNetwork(envs.single_observation_space, envs.single_action_space, cfg, net, net, "cuda", max_envs=P, max_episode_length=T)
    coll = Collector(envs, m, T)
    rows = []
    for it in range(iters + 1):   # the first iteration warms up
        torch.cuda.synchronize(); t0 = time.perf_counter()
        ln, _ = coll.collect()
        torch.cuda.synchronize(); t1 = time.perf_counter()
        m.update_from_store(coll.batch, P, it * P * T)
        torch.cuda.synchronize(); t2 = time.perf_counter()
        if it:
            rows.append((t1 - t0, t2 - t1, int(ln.max().item()) * P))
    col, upd, steps = (float(np.median([r[k] for r in rows])) for k in range(3))
    envs.close()
    return dict(envs=P, T=T, D=envs.cfg.obs_dim, collect_s=col, update_s=upd, env_steps_per_s=steps / (col + upd), collect_env_steps_per_s=steps / col)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lbf_grid_time.py measures on an H100; no CUDA device found")
    res = dict(gpu=gpu_info())
    print("GPU (name, power limit, max SM clock):", res["gpu"])
    res["env_step"] = [time_env_step(kind, E) for E in (4096, 65536) for kind in IDS]
    for r in res["env_step"]:
        print(f"env step {r['kind']:8s} (D {r['D']:3d}), {r['envs']:6d} envs: {r['us_per_launch']:7.1f} us/launch, "
              f"{r['env_steps_per_s'] / 1e6:6.1f} M env-steps/s, {r['bytes_per_env_step']} B/env-step -> {r['hbm_bytes_per_s'] / 1e9:.1f} GB/s "
              f"({100 * r['share_of_3_35_TBps']:.1f} % of 3.35 TB/s)")
    res["ia2c"] = r = time_ia2c()
    print(f"IA2C iteration on grid-2s (4096 envs, T=25, D {r['D']}): collect {r['collect_s'] * 1e3:.1f} ms, update {r['update_s'] * 1e3:.1f} ms, "
          f"{r['env_steps_per_s'] / 1e6:.2f} M env-steps/s ({r['collect_env_steps_per_s'] / 1e6:.2f} M in collection)")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "lbf_grid_time.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

"""Timings of the multi-robot warehouse path (DESIGN.md §4.7, §7b):

    python tools/rware_time.py [--out DIR]

prints the GPU's name and power limit, then
  * the env-step kernel (rware-tiny-4ag-v2, autoreset, explicit actions) per launch at 2 048 and 65 536 envs, CUDA events over 200 launches,
    with the achieved HBM bytes/s from the algorithmic byte count below and its share of the H100 SXM data sheet's 3.35 TB/s;
  * one IPPO training iteration at BASELINE.json configs[4]'s shape (2 048 envs, T = 500, 4 epochs): env-steps/s, collection and update apart;
  * the CPU oracle env on one core, for context.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_PEAK = 3.35e12   # H100 SXM data sheet


def step_bytes(cfg) -> int:
    """Algorithmic HBM bytes of one env-step: state read + written (shelf grid at its 16-byte pitch, agent words, request mask, five counters,
    episode returns), actions read, observations / rewards / flags written."""
    N, D, pitch = cfg.n_agents, cfg.obs_dim, (cfg.rows * cfg.cols + 15) // 16 * 16
    state = pitch + 4 * N + 32 + 4 * 4 + 1 + 4 * N
    return 2 * state + 4 * N + 4 * N * D + 4 * N + 2


def gpu_info() -> str:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:   # pragma: no cover
        return f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})"


def time_env_step(E: int, launches: int = 200) -> dict:
    from codebase_b200.rware import NativeRware, parse_rware_id

    cfg = parse_rware_id("rware-tiny-4ag-v2", 500)
    env = NativeRware(cfg, E, seed=1)
    env.reset()
    acts = torch.randint(0, 5, (E, cfg.n_agents), dtype=torch.int32, device="cuda")
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
    return dict(envs=E, us_per_launch=us, env_steps_per_s=E / us * 1e6, bytes_per_env_step=step_bytes(cfg), hbm_bytes_per_s=by / us * 1e6,
                share_of_3_35_TBps=by / us * 1e6 / HBM_PEAK)


def time_ippo(P: int = 2048, T: int = 500, iters: int = 2) -> dict:
    from codebase_b200.ac.model import PPONetwork
    from codebase_b200.ac.train import Collector
    from codebase_b200.utils.envs import make_env

    envs = make_env(0, name="rware:rware-tiny-4ag-v2", time_limit=T, parallel_envs=P)
    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=0.5, n_steps=10, entropy_coef=0.001, value_loss_coef=0.5,
                                target_update_interval_or_tau=0.01, standardise_returns=False, num_epochs=4, ppo_clip=0.2)
    net = types.SimpleNamespace(layers=[128, 128], parameter_sharing=False, use_rnn=False, use_orthogonal_init=True, centralised=False)
    m = PPONetwork(envs.single_observation_space, envs.single_action_space, cfg, net, net, "cuda", max_envs=P, max_episode_length=T)
    coll = Collector(envs, m, T)
    rows = []
    for it in range(iters + 1):   # the first iteration warms up
        torch.cuda.synchronize(); t0 = time.perf_counter()
        ln, _ = coll.collect()
        torch.cuda.synchronize(); t1 = time.perf_counter()
        m.update_from_store(coll.batch, P, it * P * T)
        torch.cuda.synchronize(); t2 = time.perf_counter()
        steps = int(ln.max().item()) * P
        if it:
            rows.append((t1 - t0, t2 - t1, steps))
    col, upd, steps = (float(np.median([r[k] for r in rows])) for k in range(3))
    envs.close()
    return dict(envs=P, T=T, epochs=4, collect_s=col, update_s=upd, env_steps_per_s=steps / (col + upd), collect_env_steps_per_s=steps / col)


def time_oracle(E: int = 32, steps: int = 50) -> dict:
    from codebase_b200.rware import parse_rware_id
    from oracle.rware_ref import OracleVecRware

    torch.set_num_threads(1)
    cfg = parse_rware_id("rware-tiny-4ag-v2", 500)
    v = OracleVecRware(cfg, E, seed=1)
    v.reset()
    rng = np.random.default_rng(0)
    acts = [rng.integers(0, 5, size=(E, 4)) for _ in range(steps)]
    t0 = time.perf_counter()
    for a in acts:
        v.step(a, autoreset=True)
    return dict(env_steps_per_s=E * steps / (time.perf_counter() - t0))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rware_time.py measures on an H100; no CUDA device found")
    res = dict(gpu=gpu_info())
    print("GPU (name, power limit, max SM clock):", res["gpu"])
    res["env_step"] = [time_env_step(E) for E in (2048, 65536)]
    for r in res["env_step"]:
        print(f"env step, {r['envs']} envs: {r['us_per_launch']:.1f} us/launch, {r['env_steps_per_s'] / 1e6:.1f} M env-steps/s, "
              f"{r['bytes_per_env_step']} B/env-step -> {r['hbm_bytes_per_s'] / 1e9:.1f} GB/s ({100 * r['share_of_3_35_TBps']:.1f} % of 3.35 TB/s)")
    res["ippo"] = time_ippo()
    r = res["ippo"]
    print(f"IPPO iteration (2048 envs, T=500, 4 epochs): collect {r['collect_s'] * 1e3:.0f} ms, update {r['update_s'] * 1e3:.0f} ms, "
          f"{r['env_steps_per_s'] / 1e6:.2f} M env-steps/s")
    res["oracle_cpu"] = time_oracle()
    print(f"CPU oracle, one core: {res['oracle_cpu']['env_steps_per_s']:.0f} env-steps/s")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "rware_time.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

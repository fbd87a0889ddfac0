"""Timings of the matrix-game path (DESIGN.md §4.9, §7b):

    python tools/matrix_time.py [--out DIR]

prints the GPU's name and power limit, then
  * the env-step kernel (climbing-v0, autoreset, explicit actions) per launch at 4 096, 65 536 and 1 048 576 envs, CUDA events over 200
    launches, with the achieved HBM bytes/s from the algorithmic byte count below and its share of the H100 SXM data sheet's 3.35 TB/s;
  * one IDQN iteration on climbing-v0 (4 096 envs, T = 25: the fused epsilon-greedy collection of one episode per env, then one update on a
    batch of 1 024 episodes), collection and update apart;
  * one IA2C iteration on climbing-v0 (4 096 envs, T = 25), collection and update apart.
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

NAME = "matrixgames:climbing-v0"


def step_bytes(cfg) -> int:
    """Algorithmic HBM bytes of one env-step: state read + written (previous actions, episode returns, four counters and the active flag),
    actions read, observations / rewards / flags written.  The payoff entry read per env is not counted: the table (72 B here) stays in L2."""
    N, D = cfg.n_agents, cfg.obs_dim
    state = N + 4 * N + 4 * 3 + 1
    return 2 * state + 4 * N + 4 * N * D + 4 * N + 2


def time_env_step(E: int, launches: int = 200) -> dict:
    from codebase_b200.matrix import NativeMatrix, parse_matrix_id

    cfg = parse_matrix_id(NAME, 25)
    env = NativeMatrix(cfg, E, seed=1)
    env.reset()
    acts = torch.randint(0, cfg.n_actions, (E, cfg.n_agents), dtype=torch.int32, device="cuda")
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


def _median_iteration(step, iters):
    rows = []
    for it in range(iters + 1):   # the first iteration warms up
        torch.cuda.synchronize(); t0 = time.perf_counter()
        steps = step(it, "collect")
        torch.cuda.synchronize(); t1 = time.perf_counter()
        step(it, "update")
        torch.cuda.synchronize(); t2 = time.perf_counter()
        if it:
            rows.append((t1 - t0, t2 - t1, steps))
    col, upd, steps = (float(np.median([r[k] for r in rows])) for k in range(3))
    return dict(collect_s=col, update_s=upd, env_steps_per_s=steps / (col + upd), collect_env_steps_per_s=steps / col)


def time_idqn(E: int = 4096, B: int = 1024, T: int = 25, iters: int = 5) -> dict:
    from codebase_b200.dqn.model import QNetwork
    from codebase_b200.dqn.train import Collector
    from codebase_b200.native_env import TrajStore
    from codebase_b200.utils.envs import make_env

    venv = make_env(0, name=NAME, time_limit=T, parallel_envs=E)
    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=1.0, double_q=True, target_update_interval_or_tau=200,
                                standardise_returns=False)
    model = QNetwork(venv.single_observation_space, venv.single_action_space, cfg, [128, 128], False, False, True, "cuda", max_batch=B,
                     max_episode_length=T)
    rb = TrajStore(E, venv.n_agents, T, venv.cfg.obs_dim, venv.native.device)
    coll = Collector(venv, model, T)
    idx = torch.randperm(E, device="cuda")[:B].to(torch.int32)

    def step(it, what):
        if what == "collect":
            ln, _ = coll.collect(rb, 0, 0.1)
            return int(ln.sum().item())
        model.update_from_store(rb, idx)

    res = dict(envs=E, batch=B, T=T, **_median_iteration(step, iters))
    venv.close()
    return res


def time_ia2c(P: int = 4096, T: int = 25, iters: int = 5) -> dict:
    from codebase_b200.ac.model import A2CNetwork
    from codebase_b200.ac.train import Collector
    from codebase_b200.utils.envs import make_env

    envs = make_env(0, name=NAME, time_limit=T, parallel_envs=P)
    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=0.5, n_steps=10, entropy_coef=0.001, value_loss_coef=0.5,
                                target_update_interval_or_tau=0.01, standardise_returns=False)
    net = types.SimpleNamespace(layers=[128, 128], parameter_sharing=False, use_rnn=False, use_orthogonal_init=True, centralised=False)
    m = A2CNetwork(envs.single_observation_space, envs.single_action_space, cfg, net, net, "cuda", max_envs=P, max_episode_length=T)
    coll = Collector(envs, m, T)

    def step(it, what):
        if what == "collect":
            ln, _ = coll.collect()
            return int(ln.max().item()) * P
        m.update_from_store(coll.batch, P, it * P * T)

    res = dict(envs=P, T=T, **_median_iteration(step, iters))
    envs.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("matrix_time.py measures on an H100; no CUDA device found")
    res = dict(gpu=gpu_info())
    print("GPU (name, power limit, max SM clock):", res["gpu"])
    res["env_step"] = [time_env_step(E) for E in (4096, 65536, 1048576)]
    for r in res["env_step"]:
        print(f"env step, {r['envs']} envs: {r['us_per_launch']:.1f} us/launch, {r['env_steps_per_s'] / 1e6:.1f} M env-steps/s, "
              f"{r['bytes_per_env_step']} B/env-step -> {r['hbm_bytes_per_s'] / 1e9:.1f} GB/s ({100 * r['share_of_3_35_TBps']:.1f} % of 3.35 TB/s)")
    for name, fn in (("idqn", time_idqn), ("ia2c", time_ia2c)):
        res[name] = r = fn()
        print(f"{name.upper()} iteration ({r['envs']} envs, T={r['T']}{', batch %d' % r['batch'] if 'batch' in r else ''}): "
              f"collect {r['collect_s'] * 1e3:.2f} ms, update {r['update_s'] * 1e3:.2f} ms, {r['env_steps_per_s'] / 1e6:.2f} M env-steps/s")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "matrix_time.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

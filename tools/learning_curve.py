#!/usr/bin/env python
"""Returns-curve check (BASELINE.json north_star: "returns curve matching reference within noise").

Runs IDQN on Foraging-8x8-2p-3f-v3 (time_limit 25, batch_size 128, the reference's hyper-parameters, idqn.yaml) for the
same number of environment steps and the same update : episode ratio with
  * the GPU path: E vectorised envs, E updates per iteration (codebase_b200.dqn.train pieces), S seeds;
  * the CPU restatement of the reference loop (oracle/cpu_loop.py: 1 env, one update per episode), S seeds in parallel
    on the host cores,
and prints evaluation returns (100 greedy-ish episodes, eps 0.05) at the same checkpoints as one JSON document."""
import argparse
import json
import multiprocessing as mp
import os
import sys
import time
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
TOTAL, EVAL_EVERY, B, T = 200_000, 25_000, 128, 25
HP = dict(training_start=2000, eps_start=1.0, eps_end=0.05, eps_decay_over=0.5)


def eps_at(step):
    return max(HP["eps_end"] + (HP["eps_start"] - HP["eps_end"]) * (1 - step / (TOTAL * HP["eps_decay_over"])), HP["eps_end"])


def cpu_run(seed):
    import torch

    from oracle import cpu_loop
    from oracle.lbf_ref import LBFConfig, WrappedForaging

    cfg = LBFConfig(time_limit=T)
    loop = cpu_loop.CpuIdqn(cfg, B, buffer_size=10000, seed=seed)
    eval_env = WrappedForaging(cfg, seed, env_gid=1 << 20)
    step, last_eval, curve = 0, 0, []
    while step < TOTAL + 1:
        step += loop.collect_episode(eps_at(step))
        if step > HP["training_start"] and loop.rb.pos >= B:
            loop.update()
        if step - last_eval >= EVAL_EVERY:
            rets = []
            train_env, loop.env = loop.env, eval_env
            for _ in range(100):
                obss, _ = eval_env.reset()
                done, tot = False, 0.0
                while not done:
                    obss, rew, d, tr, _ = eval_env.step(loop.act(obss, 0.05))
                    tot += sum(rew); done = d or tr
                rets.append(tot)
            loop.env = train_env
            curve.append((step, float(np.mean(rets))))
            last_eval = step
    return curve


def gpu_run(seed, E):
    import torch

    from codebase_b200.dqn.model import QNetwork
    from codebase_b200.dqn.train import Collector
    from codebase_b200.lbf import TrajStore
    from codebase_b200.utils.envs import make_env

    env = make_env(seed, name="lbforaging:Foraging-8x8-2p-3f-v3", time_limit=T, parallel_envs=E)
    eval_env = make_env(seed, name="lbforaging:Foraging-8x8-2p-3f-v3", time_limit=T, parallel_envs=100, env_gid0=1 << 30)
    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=1.0, double_q=True, target_update_interval_or_tau=200, standardise_returns=False)
    torch.manual_seed(seed)
    model = QNetwork(env.single_observation_space, env.single_action_space, cfg, [128, 128], False, False, True, "cuda", max_batch=B, max_episode_length=T)
    cap = 10000
    rb = TrajStore(cap, 2, T, 15, env.native.device)
    coll, ev = Collector(env, model, T), Collector(eval_env, model, T)
    step = pos = updates = last_eval = 0
    curve = []
    while step < TOTAL + 1:
        fl, _ = coll.collect(rb, pos % cap, eps_at(step))
        step += int(fl.sum()); pos += E
        if step > HP["training_start"] and pos >= B:
            model.update_n(rb, B, min(pos, cap), seed, updates, E)
            updates += E
        if step - last_eval >= EVAL_EVERY:
            _, ret = ev.collect(None, 0, 0.05)
            curve.append((step, float(ret.sum(1).mean())))
            last_eval = step
    return curve


def _set_budget(total, eval_every):
    global TOTAL, EVAL_EVERY
    TOTAL, EVAL_EVERY = int(total), int(eval_every)


def _cpu_entry(args):
    seed, total, eval_every = args
    _set_budget(total, eval_every)
    return cpu_run(seed)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--seeds", type=int, default=8)
    ap.add_argument("--envs", type=int, default=64)
    ap.add_argument("--total", type=int, default=TOTAL, help="environment-step budget per seed")
    ap.add_argument("--eval-every", type=int, default=EVAL_EVERY)
    ap.add_argument("--arm", default="both", choices=["both", "cpu", "gpu"],
                    help="cpu: only the CPU restatement of the reference loop (runs without a GPU); gpu: only the GPU path")
    ap.add_argument("--out", default=None, help="also write the JSON document here")
    a = ap.parse_args()
    _set_budget(a.total, a.eval_every)
    t0 = time.time()
    if a.arm != "both":
        if a.arm == "cpu":
            with mp.get_context("spawn").Pool(a.seeds) as pool:
                curves = pool.map(_cpu_entry, [(s, a.total, a.eval_every) for s in range(a.seeds)])
        else:
            curves = [gpu_run(s, a.envs) for s in range(a.seeds)]
        doc = {"what": "IDQN Foraging-8x8-2p-3f-v3, batch 128, eval returns (sum over agents, 100 episodes, eps 0.05)", "arm": a.arm, "seeds": a.seeds,
               "total_steps": a.total, "eval_every": a.eval_every, "b200_envs": a.envs if a.arm == "gpu" else None,
               "seconds": round(time.time() - t0, 1), "curves": curves}
        txt = json.dumps(doc, indent=1)
        if a.out:
            open(a.out, "w").write(txt)
        print(txt)
        sys.exit(0)
    ctx = mp.get_context("spawn")
    pool = ctx.Pool(a.seeds)
    cpu_async = pool.map_async(cpu_run, list(range(a.seeds)))
    gpu = [gpu_run(s, a.envs) for s in range(a.seeds)]
    t_gpu = time.time() - t0
    cpu = cpu_async.get()
    pool.close()
    n = min(min(len(c) for c in cpu), min(len(c) for c in gpu))
    rows = []
    for i in range(n):
        c = np.array([r[i][1] for r in cpu]); g = np.array([r[i][1] for r in gpu])
        rows.append({"env_steps~": int(np.mean([r[i][0] for r in gpu])), "reference_cpu_mean": round(float(c.mean()), 4), "reference_cpu_std": round(float(c.std()), 4),
                     "b200_mean": round(float(g.mean()), 4), "b200_std": round(float(g.std()), 4)})
    print(json.dumps({"what": "IDQN Foraging-8x8-2p-3f-v3, batch 128, eval returns (sum over agents, 100 episodes, eps 0.05)", "seeds": a.seeds, "b200_envs": a.envs,
                      "seconds_b200_all_seeds": round(t_gpu, 1), "seconds_total": round(time.time() - t0, 1), "curve": rows}, indent=1))

#!/usr/bin/env python
"""VDN / QMIX on the CPU reference loop next to the GPU runs of the same overlays (results.csv of `python -m codebase_b200.run`): idqn.yaml's
hyper-parameters (batch_size 32, training_start 2000, epsilon 1.0 -> 0.05 over half of the budget, hard target update every 200 updates),
CooperativeReward, 400 k env steps, evaluation (100 episodes at eps 0.05) and the last update's loss every 50 k steps.

The CPU arm is oracle/cpu_loop.py's one-env loop (dqn/train.py:298-311: one episode, one update) with oracle/learner_ref.py (VDN) or
oracle/qmix_ref.py (QMIX) as the learner.  CPU only:  python tools/learning_curve_mix.py --seeds 2 --out curve_mix_cpu.json"""
import argparse
import json
import multiprocessing as mp
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
B, T = 32, 25


def cpu_run(args):
    alg, seed, total, every = args
    import torch

    from oracle import cpu_loop
    from oracle import learner_ref as lr
    from oracle import qmix_ref as qr
    from oracle.lbf_ref import LBFConfig, WrappedForaging

    cfg = LBFConfig(time_limit=T, cooperative_reward=1)
    loop = cpu_loop.CpuIdqn(cfg, B, buffer_size=10000, seed=seed, hp=lr.DqnHP(mixer=1))
    if alg == "qmix":
        mix = qr.init_mixer_flat(loop.N, loop.N * loop.D, 64, 32)
        loop.st = qr.QmixState(loop.st.theta, loop.st.theta_tgt, mix, mix.clone(), loop.st.agent_net, loop.D, loop.A)
        loop.update = lambda: qr.qmix_update(loop.st, lr.batch_from_store(loop.rb.store, np.random.randint(0, len(loop.rb), size=B)), loop.hp)["loss"]
    eval_env = WrappedForaging(cfg, seed, env_gid=1 << 20)
    eps_at = lambda s: max(0.05 + 0.95 * (1 - s / (total * 0.5)), 0.05)
    step, last_eval, curve, loss, t0 = 0, 0, [], float("nan"), time.perf_counter()
    while step < total + 1:
        step += loop.collect_episode(eps_at(step))
        if step > 2000 and loop.rb.pos >= B:
            loss = loop.update()
        if step - last_eval >= every:
            rets = []
            for _ in range(100):
                obss, _ = eval_env.reset()
                done = False
                while not done:
                    obss, _, d, tr, info = eval_env.step(loop.act(obss, 0.05))
                    done = d or tr
                rets.append(float(np.sum(info["episode_returns"])))
            curve.append((step, float(np.mean(rets)), float(loss)))
            last_eval = step
    return dict(alg=alg, seed=seed, points=curve, seconds=time.perf_counter() - t0)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--seeds", type=int, default=2)
    ap.add_argument("--total", type=int, default=400_000)
    ap.add_argument("--every", type=int, default=50_000)
    ap.add_argument("--algs", default="vdn,qmix")
    ap.add_argument("--procs", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    jobs = [(alg, s, a.total, a.every) for alg in a.algs.split(",") for s in range(1, a.seeds + 1)]
    with mp.get_context("spawn").Pool(min(a.procs, len(jobs))) as pool:
        runs = pool.map(cpu_run, jobs)
    for r in runs:
        print(f"{r['alg']} seed {r['seed']}: " + " ".join(f"{s // 1000}k:{v:.3f}/loss {l:.3g}" for s, v, l in r["points"]) + f"  ({r['seconds']:.0f} s)", flush=True)
    doc = dict(what="CPU reference loop (oracle/cpu_loop.py + learner_ref / qmix_ref), evaluation return (100 episodes, eps 0.05) and the last update's loss",
               total=a.total, every=a.every, batch_size=B, runs=runs)
    if a.out:
        json.dump(doc, open(a.out, "w"), indent=1)

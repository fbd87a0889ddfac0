#!/usr/bin/env python
"""Returns curves of the actor-critic family on the CPU reference loop (oracle/cpu_loop_ac.py) next to the GPU runs of the same overlays
(the results.csv of `python -m codebase_b200.run +algorithm=<alg> ...`): same env, 64 env instances, yaml defaults, 400 k env steps,
training-episode returns logged every 51 200 steps (ac/train.py:184-186 logs the TRAINING episodes' infos).

    python tools/learning_curve_ac.py --seeds 3 --out curve_ac_cpu.json     (CPU only, ~1 min per run)"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.cpu_loop_ac import ALGS, CpuAC  # noqa: E402
from oracle.lbf_ref import LBFConfig  # noqa: E402


def run(alg, seed, total, every, envs):
    loop = CpuAC(alg, LBFConfig(), envs, seed)
    pts, last, t0 = [], -every, time.perf_counter()
    while loop.step < total + 1:
        at, ret = loop.iteration()
        if at - last >= every:
            pts.append((at, ret)); last = at
    return dict(alg=alg, seed=seed, points=pts, seconds=time.perf_counter() - t0, updates=loop.updates)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seeds", type=int, default=3)
    ap.add_argument("--total", type=int, default=400_000)
    ap.add_argument("--every", type=int, default=50_000)
    ap.add_argument("--envs", type=int, default=64)
    ap.add_argument("--algs", default=",".join(ALGS))
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    runs = []
    for alg in a.algs.split(","):
        for seed in range(1, a.seeds + 1):
            r = run(alg, seed, a.total, a.every, a.envs)
            runs.append(r)
            print(f"{alg} seed {seed}: " + " ".join(f"{s // 1000}k:{v:.3f}" for s, v in r["points"]) + f"  ({r['seconds']:.0f} s)", flush=True)
    doc = dict(what="CPU reference loop (oracle/cpu_loop_ac.py), mean training-episode return (sum over agents) of the batch logged at each checkpoint",
               envs=a.envs, total=a.total, every=a.every, runs=runs)
    table = {}
    for alg in a.algs.split(","):
        rs = [r for r in runs if r["alg"] == alg]
        n = min(len(r["points"]) for r in rs)
        table[alg] = [dict(step=int(rs[0]["points"][k][0]), mean=float(np.mean([r["points"][k][1] for r in rs])), std=float(np.std([r["points"][k][1] for r in rs])))
                      for k in range(n)]
    doc["table"] = table
    if a.out:
        json.dump(doc, open(a.out, "w"), indent=1)
    print(json.dumps(table))


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""The book's coordination comparison on the matrix games: IDQN, VDN and QMIX on climbing-nostate-v0 and penalty-100-nostate-v0, several seeds,
through `python -m codebase_b200.run` with the algorithms' own overlays (VDN and QMIX add CooperativeReward), env.time_limit = 25 and greedy
evaluation (algorithm.eps_evaluation=0).  Reports the final greedy episode return per algorithm and game (the sum over both players of the
raw payoffs: 25 x payoff of the joint action each player settles on; the optimum is 275 on climbing and 250 on penalty-100).  A report,
not a test:

    python tools/learning_curve_matrix.py [--seeds 3] [--steps 200000] [--out DIR]
"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

GAMES = ("matrixgames:climbing-nostate-v0", "matrixgames:penalty-100-nostate-v0")
ALGS = ("idqn", "vdn", "qmix")


def final_greedy_return(alg, game, seed, steps, work):
    import pandas as pd

    from codebase_b200 import run

    out = os.path.join(work, f"{alg}-{game.split(':')[-1]}-{seed}")
    run.main([f"+algorithm={alg}", f"env.name={game}", "env.time_limit=25", f"seed={seed}", f"algorithm.total_steps={steps}",
              f"algorithm.eval_interval={steps // 4}", "algorithm.eval_episodes=100", "algorithm.eps_evaluation=0.0", f"run_dir={out}"])
    df = pd.read_csv(os.path.join(out, "results.csv"))
    cols = [c for c in df.columns if c.startswith("agent") and c.endswith("/mean_episode_returns")]
    return float(df[cols].iloc[-1].sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seeds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=200_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    res = {}
    with tempfile.TemporaryDirectory() as work:
        for game in GAMES:
            for alg in ALGS:
                rets = [final_greedy_return(alg, game, s, args.steps, work) for s in range(args.seeds)]
                res[f"{game} {alg}"] = rets
                print(f"{game:38s} {alg:5s} final greedy return: mean {np.mean(rets):7.1f}  per seed {[round(r, 1) for r in rets]}", flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "learning_curve_matrix.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

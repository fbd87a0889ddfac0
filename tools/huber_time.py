"""Time one DQN-family update with the squared TD error (huber_delta = null) and with the Huber TD loss (huber_delta = 1.0), side by side, at three
shapes: bench.py's IDQN on Foraging-8x8-2p-3f (2 agents, 15 features, 6 actions; batch 1024 sampled from 4096 episodes, T = 25), QMIX on the same
shape at batch 32, and VDN on long episodes (batch 32 of 256 episodes, T = 500).  Each handle runs `update_n` (on-device replay sampling, the fused
tail) over random ragged episodes with rewards spread over [0, 4), so TD errors fall on both sides of delta; the update time is CUDA events around
`reps` updates after a warm-up, the two handles alternating over five rounds (median reported).  Prints one JSON line with the GPU's name and power
limit.

    python tools/huber_time.py [--reps 200]
"""
import argparse
import json
import os
import subprocess
import sys
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tests.helpers import random_store, space, traj_store  # noqa: E402

SHAPES = {   # name: (class, agents, features, actions, batch, episodes in the store, T)
    "idqn_foraging_8x8_2p_3f_b1024": ("QNetwork", 2, 15, 6, 1024, 4096, 25),
    "qmix_foraging_8x8_2p_3f_b32": ("QMixNetwork", 2, 15, 6, 32, 4096, 25),
    "vdn_long_T500_b32": ("VDNetwork", 2, 15, 6, 32, 256, 500),
}


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    name, power = [x.strip() for x in out.splitlines()[0].split(",")]
    return name, power


def make(cls, N, D, A, B, T, delta):
    from codebase_b200.dqn import model as M

    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=1.0, double_q=True, target_update_interval_or_tau=200,
                                standardise_returns=False, td_lambda=None, huber_delta=delta)
    args = ([space(shape=(D,))] * N, [space(n=A)] * N, cfg, [128, 128], False, False, True)
    if cls == "QMixNetwork":
        return M.QMixNetwork(*args, dict(embed_dim=64, hypernet_layers=2, hypernet_embed=32), "cuda", max_batch=B, max_episode_length=T)
    return getattr(M, cls)(*args, "cuda", max_batch=B, max_episode_length=T)


def update_ms(m, ts, B, cap, reps, first):
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0.record()
    m.update_n(ts, B, cap, 1234, first, reps)
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no GPU: this script measures on the device only")
    name, power = gpu_info()
    res = {"gpu": name, "power_limit": power, "reps": args.reps}
    for key, (cls, N, D, A, B, cap, T) in SHAPES.items():
        torch.manual_seed(0)
        ts, models = None, {}
        for mode, delta in (("squared", None), ("huber_1.0", 1.0)):
            models[mode] = make(cls, N, D, A, B, T, delta)
            if ts is None:
                s = random_store(np.random.default_rng(0), cap, N, T, D, cls != "QNetwork", A=A)
                s["rew"] *= 4.0
                ts = traj_store(s, models[mode].device)
            models[mode].update_n(ts, B, cap, 1234, 0, 20)   # warm-up
        reps = max(10, args.reps // (10 if T > 100 else 1))
        times = {mode: [] for mode in models}
        for r in range(5):
            for mode, m in models.items():
                times[mode].append(update_ms(m, ts, B, cap, reps, 20 + r * reps))
        out = {"batch": B, "T": T, "agents": N}
        for mode in models:
            out[f"{mode}_update_us"] = round(1000.0 * float(np.median(times[mode])), 2)
        out["huber_extra_us"] = round(out["huber_1.0_update_us"] - out["squared_update_us"], 2)
        res[key] = out
        for m in models.values():
            m.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

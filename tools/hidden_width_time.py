"""Time one learner update at hidden widths 32, 64 and 128 (`layers: [H, H]`) with CUDA events, on random data of the benchmark's shapes:
an IDQN update (BASELINE configs[1]: 2 agents, 15 observation features, 6 actions, batch 1024 episodes of 25 steps) and an IA2C update
(configs[2]: 8192 envs, 2 agents; 10 steps per update here).  Widths below 128 run the FP32 kernels with zero-padded 128-wide tiles; 128
runs the default (tensor-core) path.  Prints the GPU's name and power limit with the timings.

    python tools/hidden_width_time.py [--reps 50]
"""
import argparse
import os
import subprocess
import sys
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tests.helpers import ac_batch, random_store, space, traj_store  # noqa: E402

N, D, A = 2, 15, 6


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        out = f"nvidia-smi unavailable ({e})"
    return out or torch.cuda.get_device_name()


def timed(fn, reps, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / reps


def idqn_update_ms(H, reps):
    from codebase_b200.dqn import model as M

    B, T, cap = 1024, 25, 4096
    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=1.0, double_q=True, target_update_interval_or_tau=200, standardise_returns=False)
    m = M.QNetwork([space(shape=(D,))] * N, [space(n=A)] * N, cfg, [H, H], False, False, True, "cuda", max_batch=B, max_episode_length=T)
    ts = traj_store(random_store(np.random.default_rng(0), cap, N, T, D, coop=False), m.device)
    idx = torch.randint(0, cap, (B,), dtype=torch.int32, device="cuda")
    ms = timed(lambda: m.update_from_store(ts, idx), reps)
    m.close()
    return ms


def ia2c_update_ms(H, reps):
    from codebase_b200.ac import model as M

    P, T = 8192, 10
    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=0.0, n_steps=5, entropy_coef=0.001, value_loss_coef=0.5,
                                target_update_interval_or_tau=200, standardise_returns=False)
    net = types.SimpleNamespace(layers=[H, H], parameter_sharing=False, use_rnn=False, use_orthogonal_init=True, centralised=False)
    m = M.A2CNetwork([space(shape=(D,))] * N, [space(n=A)] * N, cfg, net, net, "cuda", max_envs=P, max_episode_length=T)
    ts = traj_store(ac_batch(np.random.default_rng(0), P, N, T, D, A), m.device)
    ms = timed(lambda: m.update_from_store(ts, P, 1), reps)
    m.close()
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no GPU: this script measures on the device only")
    print(f"GPU: {gpu_info()}")
    for H in (32, 64, 128):
        print(f"H={H:3d}  IDQN update {idqn_update_ms(H, args.reps):8.3f} ms   IA2C update {ia2c_update_ms(H, args.reps):8.3f} ms")


if __name__ == "__main__":
    main()

"""Time the returns kernel and the whole learner update with n-step returns and with λ-returns (algorithm.gae_lambda), side by side, at two shapes:
IA2C on Foraging-8x8-2p-3f (2 agents, 15 features, 6 actions; 8192 envs, T = 25) and IPPO on rware-tiny-4ag (4 agents, 71 features, 5 actions;
2048 envs, T = 500, 4 epochs), on random on-policy batches of those shapes.  The whole update is timed with CUDA events after a warm-up, the
n-step and λ handles alternating over three rounds (median reported); the returns kernel's time comes from a separate torch.profiler run.  Prints
one JSON line with the GPU's name and power limit.

    python tools/gae_time.py [--reps 20]
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

from tests.helpers import ac_batch, space, traj_store  # noqa: E402

SHAPES = {   # name: (class, agents, features, actions, envs, T)
    "ia2c_foraging_8x8_2p_3f": ("A2CNetwork", 2, 15, 6, 8192, 25),
    "ippo_rware_tiny_4ag": ("PPONetwork", 4, 71, 5, 2048, 500),
}


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    name, power = [x.strip() for x in out.splitlines()[0].split(",")]
    return name, power


def make(cls, N, D, A, P, T, lam):
    from codebase_b200.ac import model as M

    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=False, n_steps=5, entropy_coef=0.001, value_loss_coef=0.5,
                                target_update_interval_or_tau=200, standardise_returns=False, num_epochs=4, ppo_clip=0.2, gae_lambda=lam)
    net = types.SimpleNamespace(layers=[128, 128], parameter_sharing=False, use_rnn=False, use_orthogonal_init=True, centralised=False)
    return getattr(M, cls)([space(shape=(D,))] * N, [space(n=A)] * N, cfg, net, net, "cuda", max_envs=P, max_episode_length=T)


def update_ms(m, ts, P, reps):
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0.record()
    for _ in range(reps):
        m.update_from_store(ts, P, 1)
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / reps


def returns_kernel_us(m, ts, P, reps, kernel):
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            m.update_from_store(ts, P, 1)
        torch.cuda.synchronize()
    total, count = 0.0, 0
    for e in prof.key_averages():
        if kernel in e.key:
            total += float(getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0))
            count += int(e.count)
    if count != reps:
        raise RuntimeError(f"{kernel}: {count} launches in the profile, expected {reps}")
    return total / count


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no GPU: this script measures on the device only")
    name, power = gpu_info()
    res = {"gpu": name, "power_limit": power, "reps": args.reps}
    for key, (cls, N, D, A, P, T) in SHAPES.items():
        torch.manual_seed(0)
        ts = None
        models = {}
        for mode, lam in (("nstep", None), ("lambda", 0.95)):
            models[mode] = make(cls, N, D, A, P, T, lam)
            if ts is None:
                ts = traj_store(ac_batch(np.random.default_rng(0), P, N, T, D, A), models[mode].device)
            for _ in range(3):   # warm-up
                models[mode].update_from_store(ts, P, 1)
        reps = max(2, args.reps // (4 if cls == "PPONetwork" else 1))
        times = {"nstep": [], "lambda": []}
        for _ in range(3):
            for mode, m in models.items():
                times[mode].append(update_ms(m, ts, P, reps))
        out = {"envs": P, "T": T, "agents": N}
        for mode, kernel in (("nstep", "nstep_returns_kernel"), ("lambda", "lambda_returns_kernel")):
            out[f"{mode}_update_ms"] = round(float(np.median(times[mode])), 3)
            out[f"{mode}_returns_kernel_us"] = round(returns_kernel_us(models[mode], ts, P, reps, kernel), 2)
        res[key] = out
        for m in models.values():
            m.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

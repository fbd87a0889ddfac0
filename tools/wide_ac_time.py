"""Time of MAA2C and MAPPO (centralised critic) at a wide joint observation, Foraging-15x15-4p-5f-v3 (4 agents x 27 = 108 inputs: KP = 128 tiles,
W1 staged per tile), next to Foraging-8x8-2p-3f-v3 (2 x 15 = 30: KP = 32 tiles, W1 resident) in the same call: update time, env-steps/s of a full
iteration (collection + update), and the achieved FLOP/s of the critic's training pass (train_kernel with the critic head, from the kernel timeline;
FLOP counted from the shapes).  Prints one JSON line:  python tools/wide_ac_time.py"""
import json
import os
import sys
import time
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import gpu_info  # noqa: E402
from codebase_b200.ac import model as M  # noqa: E402
from codebase_b200.ac.train import Collector  # noqa: E402
from codebase_b200.lbf import TrajStore  # noqa: E402
from codebase_b200.utils.envs import make_env  # noqa: E402

ENVS = {"15x15-4p-5f": ("lbforaging:Foraging-15x15-4p-5f-v3", 4, 27), "8x8-2p-3f": ("lbforaging:Foraging-8x8-2p-3f-v3", 2, 15)}
A, T, E, K, EPOCHS = 6, 25, 4096, 5, 4
H = 128


def learner(alg, N, D):
    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=False, n_steps=5, entropy_coef=0.001, value_loss_coef=0.5,
                                target_update_interval_or_tau=200, standardise_returns=False, num_epochs=EPOCHS, ppo_clip=0.2)
    net = types.SimpleNamespace(layers=[128, 128], parameter_sharing=True, use_rnn=False, use_orthogonal_init=True, centralised=False)
    cnet = types.SimpleNamespace(**{**vars(net), "centralised": True})
    sp = lambda **kw: types.SimpleNamespace(shape=kw.get("shape"), n=kw.get("n"))   # noqa: E731
    cls = M.PPONetwork if alg == "mappo" else M.A2CNetwork
    return cls([sp(shape=(D,))] * N, [sp(n=A)] * N, cfg, net, cnet, "cuda", max_envs=E, max_episode_length=T)


def store(device, N, D):
    ts = TrajStore(E, N, T, D, device)
    ts.obs.copy_(torch.randint(-1, 9, ts.obs.shape, device=device).float()); ts.act.copy_(torch.randint(0, A, ts.act.shape))
    ts.rew.copy_(torch.rand_like(ts.rew)); ts.filled.fill_(1); ts.done[:, T] = 1
    return ts


def ms(fn, reps=K):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn(); torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def critic_pass_ms(m, ts, passes_per_update, reps=3):
    """ms of one critic training pass (train_kernel<KP, kHeadA2cCritic>), from the kernel timeline of `reps` updates (torch.profiler)"""
    from torch.profiler import ProfilerActivity, profile

    m.update_from_store(ts, E, 1); torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            m.update_from_store(ts, E, 1)
        torch.cuda.synchronize()
    us = sum(e.time_range.elapsed_us() for e in prof.events()
             if e.device_type == torch.autograd.DeviceType.CUDA and "train_kernel<" in e.name and ", 1>" in e.name)
    return us / 1e3 / (reps * passes_per_update)


def critic_pass_flop(N, Dc):
    """multiply-adds x 2 of the critic's training pass over every gathered row (N agents x E envs x T + 1 steps): the forward (three layers), dW3
    and dh2, dW2, dh1 (W2^T), dW1 (no input gradient)"""
    rows = N * E * (T + 1)
    fwd = H * Dc + H * H + H
    bwd = 2 * H + 2 * H * H + H * Dc
    return 2 * rows * (fwd + bwd)


def iteration_rate(alg, env_name, N, D, iters=3):
    env = make_env(0, name=env_name, time_limit=T, parallel_envs=E)
    m = learner(alg, N, D)
    col = Collector(env, m, T)
    col.collect(); m.update_from_store(col.batch, E, 0); torch.cuda.synchronize()
    t0, steps = time.perf_counter(), 0
    for i in range(iters):
        ln, _ = col.collect()
        m.update_from_store(col.batch, E, i + 1)
        steps += int(ln.max().item()) * E   # the driver's step count (ac/train.py: t * parallel_envs)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    env.close(); m.close()
    return steps / dt


def main():
    dev = torch.device("cuda", torch.cuda.current_device())
    out = dict(shape=dict(envs=E, T=T, A=A, sharing=True, n_steps=5, ppo_epochs=EPOCHS), gpu=gpu_info(torch, dev))
    for tag, (env_name, N, D) in ENVS.items():
        for alg in ("maa2c", "mappo"):
            key = f"{alg}_{tag}"
            m = learner(alg, N, D)
            ts = store(m.device, N, D)
            out[f"{key}_joint"] = N * D
            out[f"{key}_update_ms"] = ms(lambda: m.update_from_store(ts, E, 1))
            cms = critic_pass_ms(m, ts, EPOCHS if alg == "mappo" else 1)
            out[f"{key}_critic_pass_ms"] = cms
            out[f"{key}_critic_pass_tflops"] = critic_pass_flop(N, N * D) / (cms * 1e-3) / 1e12
            m.close()
            del ts
            torch.cuda.empty_cache()
            out[f"{key}_iteration_env_steps_per_s"] = iteration_rate(alg, env_name, N, D)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

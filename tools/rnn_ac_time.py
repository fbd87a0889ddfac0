"""Time of a recurrent (GRU actor + GRU critic) IA2C update at the IA2C headline shape (8192 envs x 25 steps, 2 agents, shared parameters, obs 15,
6 actions, n_steps 5), next to the MLP update of the same shape in the same call: the update split into target-critic forward, critic pass, actor
pass and tail (from the kernel timeline), env-steps/s of a full iteration (collection + update), and the
achieved FLOP/s of the recurrent passes.  Prints one JSON line:  python tools/rnn_ac_time.py"""
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

N, D, A, T, E, K = 2, 15, 6, 25, 8192, 5
H = 128
FLOP_STEP = lambda d, a: 2 * (H * d + 2 * 3 * H * H + a * H)   # noqa: E731 -- first_layer, W_ih and W_hh, final_layer: 2 x multiply-adds per row and step


def learner(use_rnn):
    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=False, n_steps=5, entropy_coef=0.001, value_loss_coef=0.5,
                                target_update_interval_or_tau=200, standardise_returns=False)
    net = types.SimpleNamespace(layers=[128, 128], parameter_sharing=True, use_rnn=use_rnn, use_orthogonal_init=True, centralised=False)
    sp = lambda **kw: types.SimpleNamespace(shape=kw.get("shape"), n=kw.get("n"))   # noqa: E731
    return M.A2CNetwork([sp(shape=(D,))] * N, [sp(n=A)] * N, cfg, net, net, "cuda", max_envs=E, max_episode_length=T)


def store(device):
    ts = TrajStore(E, N, T, D, device)
    ts.obs.copy_((torch.randint(-1, 12, ts.obs.shape, device=device) / 6.0).float()); ts.act.copy_(torch.randint(0, A, ts.act.shape))
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


def stage_split(m, ts, reps=3):
    """ms per update of (target-critic forward + n-step returns, critic pass, actor pass, tail) from the kernel timeline of `reps` recurrent updates
    (torch.profiler): the three sequence forwards of an update open the stages in stream order (target, critic, actor); the actor pass ends with its
    backward, the tail is its gradient reduction and the clip + Adam + target step"""
    from torch.profiler import ProfilerActivity, profile

    m.update_from_store(ts, E, 1); torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            m.update_from_store(ts, E, 1)
        torch.cuda.synchronize()
    kernels = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in e.name and "Memset" not in e.name),
                     key=lambda e: e.time_range.start)
    tot = dict(target=0.0, critic=0.0, actor=0.0, tail=0.0)
    stage, n_fwd = "tail", 0
    for e in kernels:
        if "gru_forward_kernel" in e.name:
            n_fwd += 1
            stage = ("target", "critic", "actor")[(n_fwd - 1) % 3]
        tot[stage] += e.time_range.elapsed_us() / 1e3
        if stage == "actor" and "gru_backward_kernel" in e.name:
            stage = "tail"
    return {k: v / reps for k, v in tot.items()}


def iteration_rate(use_rnn, iters=3):
    env = make_env(0, name="lbforaging:Foraging-8x8-2p-3f-v3", time_limit=T, parallel_envs=E)
    m = learner(use_rnn)
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
    return steps / dt, dt / iters


def main():
    dev = torch.device("cuda", torch.cuda.current_device())
    out = dict(shape=dict(alg="ia2c", envs=E, T=T, N=N, D=D, A=A, sharing=True, n_steps=5), gpu=gpu_info(torch, dev))
    for use_rnn in (True, False):
        m = learner(use_rnn)
        ts = store(m.device)
        key = "rnn" if use_rnn else "mlp"
        out[f"{key}_update_ms"] = ms(lambda: m.update_from_store(ts, E, 1))
        if use_rnn:
            split = stage_split(m, ts)
            out.update({f"rnn_{k}_ms": v for k, v in split.items()})
            rows = N * E * (T + 1)
            # the recurrent passes of one update: target-critic forward; critic and actor each a forward and a backward (~2x the forward's
            # multiply-adds: dL/dinputs and the weight gradients)
            flop = rows * (FLOP_STEP(D, 1) + 3 * FLOP_STEP(D, 1) + 3 * FLOP_STEP(D, A))
            out.update(rnn_update_gflop=flop / 1e9, rnn_passes_tflops=flop / ((split["target"] + split["critic"] + split["actor"]) * 1e-3) / 1e12)
        m.close()
        del ts
        torch.cuda.empty_cache()
        sps, it_s = iteration_rate(use_rnn)
        out[f"{key}_iteration_env_steps_per_s"], out[f"{key}_iteration_s"] = sps, it_s
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

"""Time of the recurrent (GRU) DQN training pass at the headline shape (IDQN, 1024 episodes x 25 steps, 2 agents, obs 15, 6 actions), next to the
MLP pass of the same shape, and env-steps/s of a recurrent training iteration (collection of E episodes + E updates).  Prints one JSON line:
python tools/rnn_time.py"""
import json
import os
import sys
import time
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import gpu_info  # noqa: E402
from codebase_b200.dqn import model as M  # noqa: E402
from codebase_b200.dqn.train import Collector  # noqa: E402
from codebase_b200.lbf import TrajStore  # noqa: E402
from codebase_b200.utils.envs import make_env  # noqa: E402

N, D, A, T, B, CAP, K = 2, 15, 6, 25, 1024, 4096, 50
H = 128
FLOP_ROW = 2 * (H * D + 2 * 3 * H * H + A * H)   # first_layer, W_ih and W_hh, final_layer: multiply-adds x 2 per row and step


def learner(use_rnn):
    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=1.0, double_q=True, target_update_interval_or_tau=200, standardise_returns=False)
    sp = lambda **kw: types.SimpleNamespace(shape=kw.get("shape"), n=kw.get("n"))
    return M.QNetwork([sp(shape=(D,))] * N, [sp(n=A)] * N, cfg, [128, 128], False, use_rnn, True, "cuda", max_batch=B, max_episode_length=T)


def time_updates(m):
    ts = TrajStore(CAP, N, T, D, m.device)
    ts.obs.copy_((torch.randint(-1, 12, ts.obs.shape, device=m.device) / 6.0).float()); ts.act.copy_(torch.randint(0, A, ts.act.shape))
    ts.rew.copy_(torch.rand_like(ts.rew)); ts.filled.fill_(1)
    m.update_n(ts, B, CAP, 1, 0, 5)
    torch.cuda.synchronize()
    m.timing(True)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); m.update_n(ts, B, CAP, 1, 5, K); e1.record()
    torch.cuda.synchronize()
    pass_ms, n = m.timing(False)
    return pass_ms / max(n, 1), e0.elapsed_time(e1) / K


def iteration_rate(E=1024, iters=3):
    env = make_env(0, name="lbforaging:Foraging-8x8-2p-3f-v3", time_limit=T, parallel_envs=E)
    m = learner(True)
    rb = TrajStore(CAP, env.n_agents, T, env.cfg.obs_dim, env.native.device)
    col = Collector(env, m, T)
    pos = 0
    for _ in range(CAP // E):   # fill the ring once
        col.collect(rb, pos % CAP, 1.0); pos += E
    torch.cuda.synchronize()
    t0, steps = time.perf_counter(), 0
    for i in range(iters):
        ln, _ = col.collect(rb, pos % CAP, 0.5); pos += E
        steps += int(ln.sum().item())
        m.update_n(rb, B, CAP, 1, 1000 + i * E, E)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    env.close(); m.close()
    return steps / dt, dt / iters


def main():
    rnn_pass, rnn_update = time_updates(learner(True))
    mlp_pass, mlp_update = time_updates(learner(False))
    rows = N * B * (T + 1)
    flop_pass = 3 * rows * FLOP_ROW   # online forward + backward (twice the forward's multiply-adds) of the timed window
    sps, it_s = iteration_rate()
    out = dict(shape=dict(alg="idqn", B=B, T=T, N=N, D=D, A=A), gpu=gpu_info(torch, torch.device("cuda", torch.cuda.current_device())),
               rnn_pass_ms=rnn_pass, rnn_update_ms=rnn_update, mlp_pass_ms=mlp_pass, mlp_update_ms=mlp_update,
               rnn_flop_per_row_forward=FLOP_ROW, rnn_pass_gflop=flop_pass / 1e9, rnn_pass_tflops=flop_pass / (rnn_pass * 1e-3) / 1e12,
               rnn_iteration_env_steps_per_s=sps, rnn_iteration_s=it_s)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

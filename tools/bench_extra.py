#!/usr/bin/env python
"""Secondary measurements quoted in DESIGN.md / profiles (not bench.py's contract):
  * lbf_step_kernel alone against its HBM roofline (322 B per env-step at 8x8-2p-3f, SURVEY §8d) for a sweep of env counts;
  * the fused rollout (forward + eps-greedy + transition + replay write) in env-steps/s;
  * IA2C (BASELINE.json configs[2]: 8192 envs, parameter sharing, n_steps=5) iteration throughput.
CUDA events on the launching stream, >= 3 warm-up launches, JSON lines on stdout."""
import json
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from codebase_b200.ac.model import A2CNetwork  # noqa: E402
from codebase_b200.ac.train import Collector as ACCollector  # noqa: E402
from codebase_b200.dqn.model import QNetwork  # noqa: E402
from codebase_b200.dqn.train import Collector  # noqa: E402
from codebase_b200.lbf import LbfConfig, NativeLbf, TrajStore  # noqa: E402
from codebase_b200.utils.envs import make_env  # noqa: E402

PEAKS = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else {}
HBM = PEAKS.get("hbm_gbs", 6650.0)


def timed(fn, iters, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters  # ms


def env_sweep():
    for name, kw, bytes_per_step in (("8x8-2p-3f", {}, 322), ("15x15-4p-5f", dict(rows=15, cols=15, n_agents=4, max_num_food=5, sight=15), 1004)):
        for E in (4096, 65536, 1 << 20):
            env = NativeLbf(LbfConfig(**kw), E, seed=1)
            env.reset()
            acts = torch.randint(0, 6, (E, env.N), dtype=torch.int32, device="cuda")
            ms = timed(lambda: env.step(acts, autoreset=True), 50)
            gbs = E * bytes_per_step / (ms / 1e3) / 1e9
            print(json.dumps({"kernel": "lbf_step_kernel", "config": name, "n_envs": E, "us_per_launch": 1e3 * ms, "env_steps_per_s": E / (ms / 1e3),
                              "algorithmic_bytes_per_step": bytes_per_step, "achieved_gbs": gbs, "hbm_peak_gbs": HBM, "frac": gbs / HBM}))
            env.close()


def rollout():
    for E in (4096, 65536):
        env = make_env(0, name="lbforaging:Foraging-8x8-2p-3f-v3", time_limit=25, parallel_envs=E)
        cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=1.0, double_q=True, target_update_interval_or_tau=200, standardise_returns=False)
        model = QNetwork(env.single_observation_space, env.single_action_space, cfg, [128, 128], False, False, True, "cuda", max_batch=32, max_episode_length=25)
        rb = TrajStore(E, 2, 25, 15, env.native.device)
        coll = Collector(env, model, 25)
        ms = timed(lambda: coll.collect(rb, 0, 0.3), 10)
        steps = int(env.native.final_len.sum())
        print(json.dumps({"what": "fused IDQN rollout (25 x [mlp_forward + lbf rollout_step] + reset), no learner", "n_envs": E, "ms_per_iteration": ms,
                          "env_steps_per_s": steps / (ms / 1e3)}))


def ia2c():
    P = 8192
    env = make_env(0, name="lbforaging:Foraging-8x8-2p-3f-v3", time_limit=25, parallel_envs=P)
    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=False, n_steps=5, entropy_coef=0.001, value_loss_coef=0.5,
                                target_update_interval_or_tau=200, standardise_returns=False)
    net = types.SimpleNamespace(layers=[128, 128], parameter_sharing=True, use_rnn=False, use_orthogonal_init=True, centralised=False)
    model = A2CNetwork(env.single_observation_space, env.single_action_space, cfg, net, net, "cuda", max_envs=P, max_episode_length=25)
    coll = ACCollector(env, model, 25)
    state = {"step": 0}

    def it():
        coll.collect()
        model.update_from_store(coll.batch, P, state["step"])
        state["step"] += 25 * P

    ms = timed(it, 10)
    steps = int(env.native.final_len.sum())
    rows = 2 * 26 * P
    flop = (1 + 3 + 3) * rows * 2 * (15 * 128 + 128 * 128 + 128 * 6)  # target critic fwd + critic fwd/bwd + actor fwd/bwd (approx., actor width)
    ms_upd = timed(lambda: model.update_from_store(coll.batch, P, 0), 10)
    print(json.dumps({"what": "IA2C iteration, BASELINE configs[2]: 8192 envs, full parameter sharing, n_steps=5 (collect one episode per env + one update)",
                      "ms_per_iteration": ms, "env_steps_per_s": steps / (ms / 1e3), "ms_per_update": ms_upd, "update_tflops": flop / (ms_upd / 1e3) / 1e12}))


if __name__ == "__main__":
    torch.cuda.set_device(0)
    which = sys.argv[1:] or ["env_sweep", "rollout", "ia2c"]   # e.g. `python tools/bench_extra.py env_sweep` (the ncu capture of lbf_step_kernel)
    for name in which:
        {"env_sweep": env_sweep, "rollout": rollout, "ia2c": ia2c}[name]()

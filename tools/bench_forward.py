#!/usr/bin/env python
"""Forward-only pass timing: wgmma (3xTF32) vs FP32 FFMA kernels on the row count of one IDQN target pass
(B=1024 episodes x 26 steps x 2 agents = 53 248 rows).  CUDA events, warm; JSON lines."""
import ctypes as C
import json
import os
import sys
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from codebase_b200 import _native as nat  # noqa: E402
from codebase_b200.dqn.model import QNetwork  # noqa: E402


def main():
    torch.cuda.set_device(0)
    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=1.0, double_q=True, target_update_interval_or_tau=200, standardise_returns=False)
    sp = lambda **k: types.SimpleNamespace(shape=k.get("shape"), n=k.get("n"))
    m = QNetwork([sp(shape=(15,))] * 2, [sp(n=6)] * 2, cfg, [128, 128], False, False, True, "cuda", max_batch=8, max_episode_length=25)
    for E in (4096, 26624, 262144):
        obs = torch.randint(-1, 8, (E, 2, 15), device="cuda").float()
        out = torch.empty(E, 2, 6, device="cuda")
        for tc in (1, 0):
            nat.check(nat.lib().marl_set_option(b"tensor_core_forward", C.c_int32(tc)), "opt")
            for _ in range(5):
                m.q_values(obs, out=out)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(50):
                m.q_values(obs, out=out)
            e1.record(); torch.cuda.synchronize()
            us = e0.elapsed_time(e1) / 50 * 1e3
            flop = E * 2 * 38144
            print(json.dumps({"rows": 2 * E, "impl": "wgmma_3xtf32" if tc else "ffma_fp32", "us_per_pass_incl_pack": us, "tflops_fp32_equiv": flop / us / 1e6}))


if __name__ == "__main__":
    main()

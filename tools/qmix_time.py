"""Time of one QMIX update (update_n, batch 1024 episodes x T 25) for both hypernetwork forms and standardise_returns off / on, at
Foraging-8x8-2p-3f (2 agents, obs 15) and Foraging-15x15-4p-5f (4 agents, obs 27), next to VDN at the first shape:  python tools/qmix_time.py
Prints the card's name and power limit with the numbers.  The episodes are random (no learnable structure): with one-layer hypernetworks and
standardise_returns the reference's own arithmetic (restated in tests/qmix_options_ref.py) drives the loss to NaN within ~20 updates there, which the output says.
FP32 arithmetic runs at the same speed on NaN operands."""
import os
import subprocess
import sys
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from codebase_b200.dqn import model as M  # noqa: E402
from codebase_b200.lbf import TrajStore  # noqa: E402

A, T, B, CAP, WARM, TIMED = 6, 25, 1024, 4096, 20, 200


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name() + ", power limit not read"


def time_one(cls, N, D, mixing=None, standardise=False):
    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=1.0, double_q=True, target_update_interval_or_tau=200,
                                standardise_returns=standardise)
    sp = lambda **kw: types.SimpleNamespace(shape=kw.get("shape"), n=kw.get("n"))
    args = [[sp(shape=(D,))] * N, [sp(n=A)] * N, cfg, [128, 128], False, False, True] + ([mixing] if mixing else [])
    m = cls(*args, "cuda", max_batch=B, max_episode_length=T)
    ts = TrajStore(CAP, N, T, D, m.device)
    ts.obs.copy_(torch.randn_like(ts.obs)); ts.act.copy_(torch.randint(0, A, ts.act.shape)); ts.rew.copy_(torch.rand_like(ts.rew).mean(1, keepdim=True).expand_as(ts.rew))
    ts.filled.fill_(1)
    m.update_n(ts, B, CAP, 1, 0, WARM)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); m.update_n(ts, B, CAP, 1, WARM, TIMED); e1.record(); torch.cuda.synchronize()
    finite = bool(torch.isfinite(m._metrics[0]))
    m.close()
    return e0.elapsed_time(e1) / TIMED * 1e3, finite


def main():
    print(f"card: {card()}", flush=True)
    print(f"vdn 8x8-2p-3f (N 2, D 15): {time_one(M.VDNetwork, 2, 15)[0]:.1f} us per update (batch {B} x T {T})", flush=True)
    for env, N, D in (("8x8-2p-3f", 2, 15), ("15x15-4p-5f", 4, 27)):
        for hl in (2, 1):
            for std in (False, True):
                us, finite = time_one(M.QMixNetwork, N, D, dict(embed_dim=64, hypernet_layers=hl, hypernet_embed=32), std)
                print(f"qmix {env} (N {N}, D {D}) hypernet_layers {hl} standardise_returns {std}: {us:.1f} us per update (batch {B} x T {T})"
                      f"{'' if finite else ', loss went non-finite on the synthetic data'}", flush=True)


if __name__ == "__main__":
    main()

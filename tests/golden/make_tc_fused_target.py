"""Generates tests/golden/tc_fused_target.npz on a GPU: what the DQN tensor-core training pass computes, bit for bit, for the learners with an
external TD head -- QMIX, and IDQN and VDN with standardise_returns.  Per case: one pass's gradient sums and loss statistics (update_grads; QMIX:
the mixer's too), and the parameters after three updates of the multi-update path (update_n).  The training forward kernel computes the target
network's outputs (and for these learners the online outputs the TD head reads) on the rows it already holds, where separate forward kernels
computed them before; tests/test_tc_fused_target_gpu.py holds it to the numbers of those separate forwards.
    python tests/golden/make_tc_fused_target.py [OUT.npz]"""
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from tests.helpers import random_store, space  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "tc_fused_target.npz")
A, CAP, UPDATES, SAMPLE_SEED = 6, 300, 3, 78
# name: (mixer, N, D, T, B, parameter sharing, standardise_returns, seed).  QMIX with shared agents; IDQN with standardise_returns at the
# benchmark's shape; VDN with standardise_returns at a wider observation and a batch whose CTAs end in partial tiles.
CASES = {
    "qmix": (2, 3, 15, 25, 256, True, False, 44),
    "idqn_std": (0, 2, 15, 25, 1024, False, True, 55),
    "vdn_std": (1, 4, 27, 25, 333, True, True, 66),
}


def _model(case):
    import torch

    from codebase_b200.dqn import model as M

    mixer, N, D, T, B, sharing, std, seed = CASES[case]
    torch.manual_seed(seed)
    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=1.0, double_q=True, target_update_interval_or_tau=200, standardise_returns=std)
    obs, acts = [space(shape=(D,))] * N, [space(n=A)] * N
    if mixer == 2:
        m = M.QMixNetwork(obs, acts, cfg, [128, 128], sharing, False, True, dict(embed_dim=32, hypernet_layers=2, hypernet_embed=64), "cuda",
                          max_batch=B, max_episode_length=T)
    else:
        m = (M.VDNetwork if mixer else M.QNetwork)(obs, acts, cfg, [128, 128], sharing, False, True, "cuda", max_batch=B, max_episode_length=T)
    rng = np.random.default_rng(seed)
    noise = lambda s_: torch.as_tensor(s_ * rng.standard_normal(m.theta.numel()), dtype=torch.float32).to(m.theta.device).view_as(m.theta)
    m.theta.add_(noise(0.02)); m.hard_update(); m.theta.add_(noise(0.01)); m.params_changed()   # online and target networks differ
    return m, rng


def run_case(case):
    """{grad: gradient sums | loss numerator | filled count | spare, theta: parameters after UPDATES updates, metrics: their loss statistics;
    QMIX also mix_grad and mix: the mixer's}"""
    import torch

    from codebase_b200.lbf import TrajStore

    mixer, N, D, T, B, _, _, _ = CASES[case]
    m, rng = _model(case)
    s = random_store(rng, CAP, N, T, D, bool(mixer))
    idx = rng.integers(0, CAP, size=B).astype(np.int32)
    ts = TrajStore(CAP, N, T, D, m.device)
    for k in ("obs", "act", "rew", "done", "filled"):
        getattr(ts, k).copy_(torch.as_tensor(s[k]))
    m.update_grads(ts, torch.tensor(idx, device="cuda"))
    torch.cuda.synchronize()
    out = {"grad": m.grad.cpu().numpy().copy()}
    if mixer == 2:
        out["mix_grad"] = m.mix_grad.cpu().numpy().copy()
    m2, _ = _model(case)
    met = m2.update_n(ts, B, CAP, SAMPLE_SEED, 0, UPDATES)
    torch.cuda.synchronize()
    out["theta"] = m2.theta.cpu().numpy().copy()
    out["metrics"] = met.cpu().numpy().copy()
    if mixer == 2:
        out["mix"] = m2.mix.cpu().numpy().copy()
    return out


if __name__ == "__main__":
    out = sys.argv[1] if len(sys.argv) > 1 else OUT
    arrays = {}
    for case in CASES:
        for k, v in run_case(case).items():
            arrays[f"{case}.{k}"] = v
    np.savez_compressed(out, **arrays)
    print("wrote", out, {k: v.shape for k, v in arrays.items()})

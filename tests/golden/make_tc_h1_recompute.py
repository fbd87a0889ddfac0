"""Generates tests/golden/tc_h1_recompute.npz on a GPU: what the DQN tensor-core training pass (tc_train.cu) computes, bit for bit, for three
seeded cases -- one pass's per-CTA-reduced gradient sums and loss statistics (update_grads), and the parameters after three updates of the
multi-update path (update_n).  The weight-gradient kernel rebuilds H1 from the gathered observation rows instead of reading back a stored copy;
tests/test_tc_h1_recompute_gpu.py holds it to the numbers of the pass that stored H1.
    python tests/golden/make_tc_h1_recompute.py [OUT.npz]"""
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from tests.helpers import random_store, space  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "tc_h1_recompute.npz")
A, CAP, UPDATES, SAMPLE_SEED = 6, 300, 3, 77
# name: (mixer, N, D, T, B, parameter sharing, seed).  The benchmark's IDQN shape; VDN at a wider observation; a ragged case whose CTAs end in
# partial tiles and chunks, with two networks for three agents.
CASES = {
    "idqn_bench": (0, 2, 15, 25, 1024, False, 11),
    "vdn_d27": (1, 4, 27, 25, 256, True, 22),
    "ragged": (0, 3, 15, 7, 333, [0, 1, 0], 33),
}


def _model(case):
    import torch

    from codebase_b200.dqn import model as M

    mixer, N, D, T, B, sharing, seed = CASES[case]
    torch.manual_seed(seed)
    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=1.0, double_q=True, target_update_interval_or_tau=200, standardise_returns=False)
    m = (M.VDNetwork if mixer else M.QNetwork)([space(shape=(D,))] * N, [space(n=A)] * N, cfg, [128, 128], sharing, False, True, "cuda", max_batch=B, max_episode_length=T)
    rng = np.random.default_rng(seed)
    noise = lambda s_: torch.as_tensor(s_ * rng.standard_normal(m.theta.numel()), dtype=torch.float32).to(m.theta.device).view_as(m.theta)
    m.theta.add_(noise(0.02)); m.hard_update(); m.theta.add_(noise(0.01)); m.params_changed()   # online and target networks differ
    return m, rng


def run_case(case):
    """{grad: gradient sums | loss numerator | filled count | spare, theta: parameters after UPDATES updates, metrics: their loss statistics}"""
    import torch

    from codebase_b200.lbf import TrajStore

    mixer, N, D, T, B, _, _ = CASES[case]
    m, rng = _model(case)
    s = random_store(rng, CAP, N, T, D, bool(mixer))
    idx = rng.integers(0, CAP, size=B).astype(np.int32)
    ts = TrajStore(CAP, N, T, D, m.device)
    for k in ("obs", "act", "rew", "done", "filled"):
        getattr(ts, k).copy_(torch.as_tensor(s[k]))
    m.update_grads(ts, torch.tensor(idx, device="cuda"))
    torch.cuda.synchronize()
    grad = m.grad.cpu().numpy().copy()
    m2, _ = _model(case)
    met = m2.update_n(ts, B, CAP, SAMPLE_SEED, 0, UPDATES)
    torch.cuda.synchronize()
    return {"grad": grad, "theta": m2.theta.cpu().numpy().copy(), "metrics": met.cpu().numpy().copy()}


if __name__ == "__main__":
    out = sys.argv[1] if len(sys.argv) > 1 else OUT
    arrays = {}
    for case in CASES:
        for k, v in run_case(case).items():
            arrays[f"{case}.{k}"] = v
    np.savez_compressed(out, **arrays)
    print("wrote", out, {k: v.shape for k, v in arrays.items()})

"""Generates tests/golden/tc_h2_layout.npz on a GPU: what the DQN tensor-core training pass (tc_train.cu) computes, bit for bit, across the
learners, observation widths, network counts and row splits the pass distinguishes -- one pass's gradient sums and loss statistics
(update_grads; QMIX: the mixer's too), and the parameters after three updates of the multi-update path (update_n) with their loss statistics.
The training forward stores H2 in its accumulator-fragment order, one slab of 64-row tiles per CTA, and the weight-gradient kernel stages its
chunks from that order; tests/test_tc_h2_layout_gpu.py holds them to the numbers of the pass that stored H2 feature-major.
The fixture keeps, per array, the SHA-256 of its float32 bytes (the bit-identity check) and every SAMPLE_STRIDE-th value (to say where and by
how much a mismatch differs), not the arrays themselves: half a million values over the six cases.
    python tests/golden/make_tc_h2_layout.py [OUT.npz]"""
import hashlib
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from tests.helpers import random_store, space  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "tc_h2_layout.npz")
A, CAP, UPDATES, SAMPLE_SEED = 6, 300, 3, 79
SAMPLE_STRIDE = 61
# name: (mixer, N, D, T, B, parameter sharing, standardise_returns, seed).  D runs over 1, 8, 9, 15, 27 and 31 (one to four k-steps of layer 1),
# the networks over one to four.  Rows per CTA on a 132-SM H100 (episodes of T + 1 rows, split evenly over the CTAs of a network):
#   idqn_d1_one_chunk  one CTA of 21 rows: a single, partial chunk
#   idqn_d8_4nets      546 or 572 rows: nine tiles (odd), the last one partial
#   vdn_d9_2nets       55 or 66 rows: one partial tile, or a full one and a second of two rows
#   idqn_std_d15       the benchmark's shape with standardise_returns: 390 or 416 rows, seven tiles (odd), the last one partial
#   qmix_d27_3nets     52 or 78 rows: one or two tiles, partial
#   idqn_d31_shared    56 or 64 rows: one tile, partial or full
CASES = {
    "idqn_d1_one_chunk": (0, 1, 1, 20, 1, False, False, 101),
    "idqn_d8_4nets": (0, 4, 8, 25, 700, False, False, 102),
    "vdn_d9_2nets": (1, 2, 9, 10, 256, False, False, 103),
    "idqn_std_d15": (0, 2, 15, 25, 1024, False, True, 104),
    "qmix_d27_3nets": (2, 3, 27, 25, 128, False, False, 105),
    "idqn_d31_shared": (0, 3, 31, 7, 333, True, False, 106),
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


def fingerprint(v):
    """{sha256: SHA-256 of the float32 bytes (uint8[32]), size, sample: every SAMPLE_STRIDE-th value} of one array"""
    v = np.ascontiguousarray(v, dtype=np.float32)
    return {"sha256": np.frombuffer(hashlib.sha256(v.tobytes()).digest(), np.uint8).copy(), "size": np.int64(v.size), "sample": v[::SAMPLE_STRIDE].copy()}


if __name__ == "__main__":
    out = sys.argv[1] if len(sys.argv) > 1 else OUT
    arrays = {}
    for case in CASES:
        for k, v in run_case(case).items():
            for f, x in fingerprint(v).items():
                arrays[f"{case}.{k}.{f}"] = x
    np.savez_compressed(out, **arrays)
    print("wrote", out, {k: v.shape for k, v in arrays.items()})

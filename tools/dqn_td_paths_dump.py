"""Run a few seeded `update_n` calls through every TD-head path of the DQN family and save what they computed, so that two builds of the
library can be compared bit for bit (`--compare`).  Only the public Python API is used, so the same script runs against an older build
(MARL_B200_SO=<path of that build's libmarlb200.so>).

Paths: IDQN and VDN on the tensor-core pipeline (plain and standardise_returns), the recurrent pass (IDQN plain and standardised, VDN), QMIX with
one and two hypernetwork layers (plain and standardised), IDQN at layers [64, 64] (the FP32 training kernel's own head, double-Q and max),
IDQN at 128 with tensor_core_backward=0, and VDN with tensor_core_forward=0 (the external head after a target forward of its own).  TD(λ)
targets (algorithm.td_lambda) for IDQN, recurrent IDQN, VDN and QMIX with one and two hypernetwork layers, each plain and standardised, and the
Huber TD loss (algorithm.huber_delta) for IDQN, recurrent IDQN, VDN and QMIX.  Per case: theta, theta_tgt, adam_m, adam_v, the metrics of the
last update and (standardise_returns) the RunningMeanStd statistics; QMIX also the mixer's parameters.

    python tools/dqn_td_paths_dump.py OUT.npz [--updates 4]
    python tools/dqn_td_paths_dump.py --compare A.npz B.npz
"""
import argparse
import collections
import ctypes as C
import os
import subprocess
import sys
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tests.helpers import random_store, space, traj_store  # noqa: E402

N, D, A, T, CAP, B = 3, 15, 6, 25, 512, 128
MIXING = {1: dict(embed_dim=32, hypernet_layers=1, hypernet_embed=64), 2: dict(embed_dim=32, hypernet_layers=2, hypernet_embed=64)}

# cls: learner class; H: hidden width; hl: QMIX's hypernetwork layers; tc_bwd / tc_fwd: the process-wide tensor_core_backward / _forward options
Case = collections.namedtuple("Case", "cls H rnn std double_q hl tc_bwd tc_fwd td_lambda huber_delta",
                              defaults=(128, False, False, True, 0, 1, 1, None, None))
LAM, HUBER = 0.8, 0.5
CASES = {
    "idqn": Case("QNetwork"),
    "idqn_std": Case("QNetwork", std=True),
    "vdn": Case("VDNetwork"),
    "vdn_std": Case("VDNetwork", std=True),
    "vdn_maxq": Case("VDNetwork", double_q=False),
    "rnn_idqn": Case("QNetwork", rnn=True),
    "rnn_idqn_std": Case("QNetwork", rnn=True, std=True),
    "rnn_vdn": Case("VDNetwork", rnn=True),
    "qmix_hl1": Case("QMixNetwork", hl=1),
    "qmix_hl2": Case("QMixNetwork", hl=2),
    "qmix_hl1_std": Case("QMixNetwork", std=True, hl=1),
    "qmix_hl2_std": Case("QMixNetwork", std=True, hl=2),
    "idqn_h64": Case("QNetwork", H=64),
    "idqn_h64_maxq": Case("QNetwork", H=64, double_q=False),
    "idqn_tcbwd0": Case("QNetwork", tc_bwd=0),
    "vdn_tcfwd0": Case("VDNetwork", tc_fwd=0),
    **{f"{name}_lam{'_std' if std else ''}": Case(cls, rnn=rnn, std=std, hl=hl, td_lambda=LAM)
       for name, cls, rnn, hl in (("idqn", "QNetwork", False, 0), ("rnn_idqn", "QNetwork", True, 0), ("vdn", "VDNetwork", False, 0),
                                  ("qmix_hl1", "QMixNetwork", False, 1), ("qmix_hl2", "QMixNetwork", False, 2))
       for std in (False, True)},
    "idqn_huber": Case("QNetwork", huber_delta=HUBER),
    "rnn_idqn_huber": Case("QNetwork", rnn=True, huber_delta=HUBER),
    "vdn_huber": Case("VDNetwork", huber_delta=HUBER),
    "qmix_hl2_huber": Case("QMixNetwork", hl=2, huber_delta=HUBER),
}


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        out = f"nvidia-smi unavailable ({e})"
    return out or torch.cuda.get_device_name()


def set_option(name, on):
    from codebase_b200 import _native as nat

    nat.check(nat.lib().marl_set_option(name, C.c_int32(int(on))), "marl_set_option")


def run_case(name, n_updates):
    from codebase_b200.dqn import model as M

    c = CASES[name]
    torch.manual_seed(1)
    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=1.0, double_q=c.double_q, target_update_interval_or_tau=2,
                                standardise_returns=c.std, td_lambda=c.td_lambda, huber_delta=c.huber_delta)
    set_option(b"tensor_core_backward", c.tc_bwd)
    set_option(b"tensor_core_forward", c.tc_fwd)
    try:
        args = ([space(shape=(D,))] * N, [space(n=A)] * N, cfg, [c.H, c.H], False, c.rnn, True)
        if c.cls == "QMixNetwork":
            m = M.QMixNetwork(*args, MIXING[c.hl], "cuda", max_batch=B, max_episode_length=T)
        else:
            m = getattr(M, c.cls)(*args, "cuda", max_batch=B, max_episode_length=T)
        s = random_store(np.random.default_rng(2), CAP, N, T, D, coop=c.cls != "QNetwork", A=A)
        s["obs"] = (s["obs"] / 6.0).astype(np.float32)
        ts = traj_store(s, m.device)
        metrics = m.update_n(ts, B, CAP, seed=7, first_update_idx=0, n_updates=n_updates)
        torch.cuda.synchronize()
    finally:
        set_option(b"tensor_core_backward", 1)
        set_option(b"tensor_core_forward", 1)
    out = {k: getattr(m, k).detach().cpu().numpy().copy() for k in ("theta", "theta_tgt", "adam_m", "adam_v")}
    out["metrics"] = metrics.detach().cpu().numpy().copy()
    if c.std:
        mean, var, count = m.ret_ms()
        out["ret_ms"] = np.concatenate([mean.numpy(), var.numpy()])
        out["ret_count"] = np.array([count])
    if c.cls == "QMixNetwork":
        out["mix"] = m.mix.detach().cpu().numpy().copy()
        out["mix_tgt"] = m.mix_tgt.detach().cpu().numpy().copy()
    m.close()
    return out


def compare(a_path, b_path):
    a, b = np.load(a_path), np.load(b_path)
    bad = sorted(set(a.files) ^ set(b.files))
    for k in sorted(set(a.files) & set(b.files)):
        same = a[k].dtype == b[k].dtype and a[k].shape == b[k].shape and a[k].tobytes() == b[k].tobytes()
        if not same:
            bad.append(k)
    print(f"{len(set(a.files) & set(b.files))} arrays compared, {len(bad)} differ" + (": " + ", ".join(bad) if bad else " (bit-identical)"))
    return 1 if bad else 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out", nargs="?")
    ap.add_argument("--updates", type=int, default=4)
    ap.add_argument("--compare", nargs=2, metavar=("A", "B"))
    args = ap.parse_args()
    if args.compare:
        sys.exit(compare(*args.compare))
    if not args.out:
        ap.error("OUT.npz is required")
    if not torch.cuda.is_available():
        sys.exit("no GPU: this script runs the device kernels only")
    print(f"GPU: {gpu_info()}")
    arrays = {}
    for name in CASES:
        for k, v in run_case(name, args.updates).items():
            arrays[f"{name}.{k}"] = v
        print(f"{name}: loss {arrays[f'{name}.metrics'][0]:.6g}")
    np.savez(args.out, **arrays)


if __name__ == "__main__":
    main()

"""Run a few seeded `update_n` calls through every TD-head path of the DQN family and save what they computed, so that two builds of the
library can be compared bit for bit (`--compare`).  Only the public Python API is used, so the same script runs against an older build
(MARL_B200_SO=<path of that build's libmarlb200.so>).

Paths: IDQN and VDN on the tensor-core pipeline (plain and standardise_returns), the recurrent pass (IDQN plain and standardised, VDN), QMIX with
one and two hypernetwork layers (plain and standardised), IDQN at layers [64, 64] (the FP32 training kernel's own head, double-Q and max), and
IDQN at 128 with tensor_core_backward=0.  Per case: theta, theta_tgt, adam_m, adam_v, the metrics of the last update and (standardise_returns)
the RunningMeanStd statistics; QMIX also the mixer's parameters.

    python tools/dqn_td_paths_dump.py OUT.npz [--updates 4]
    python tools/dqn_td_paths_dump.py --compare A.npz B.npz
"""
import argparse
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

# name: (learner class, layers, use_rnn, standardise_returns, double_q, hypernet_layers, tensor_core_backward)
CASES = {
    "idqn": ("QNetwork", 128, False, False, True, 0, 1),
    "idqn_std": ("QNetwork", 128, False, True, True, 0, 1),
    "vdn": ("VDNetwork", 128, False, False, True, 0, 1),
    "vdn_std": ("VDNetwork", 128, False, True, True, 0, 1),
    "vdn_maxq": ("VDNetwork", 128, False, False, False, 0, 1),
    "rnn_idqn": ("QNetwork", 128, True, False, True, 0, 1),
    "rnn_idqn_std": ("QNetwork", 128, True, True, True, 0, 1),
    "rnn_vdn": ("VDNetwork", 128, True, False, True, 0, 1),
    "qmix_hl1": ("QMixNetwork", 128, False, False, True, 1, 1),
    "qmix_hl2": ("QMixNetwork", 128, False, False, True, 2, 1),
    "qmix_hl1_std": ("QMixNetwork", 128, False, True, True, 1, 1),
    "qmix_hl2_std": ("QMixNetwork", 128, False, True, True, 2, 1),
    "idqn_h64": ("QNetwork", 64, False, False, True, 0, 1),
    "idqn_h64_maxq": ("QNetwork", 64, False, False, False, 0, 1),
    "idqn_tcbwd0": ("QNetwork", 128, False, False, True, 0, 0),
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

    cls, H, rnn, std, double_q, hl, tc_bwd = CASES[name]
    torch.manual_seed(1)
    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=1.0, double_q=double_q, target_update_interval_or_tau=2,
                                standardise_returns=std)
    args = ([space(shape=(D,))] * N, [space(n=A)] * N, cfg, [H, H], False, rnn, True)
    if cls == "QMixNetwork":
        m = M.QMixNetwork(*args, MIXING[hl], "cuda", max_batch=B, max_episode_length=T)
    else:
        m = getattr(M, cls)(*args, "cuda", max_batch=B, max_episode_length=T)
    s = random_store(np.random.default_rng(2), CAP, N, T, D, coop=cls != "QNetwork", A=A)
    s["obs"] = (s["obs"] / 6.0).astype(np.float32)
    ts = traj_store(s, m.device)
    set_option(b"tensor_core_backward", tc_bwd)
    try:
        metrics = m.update_n(ts, B, CAP, seed=7, first_update_idx=0, n_updates=n_updates)
        torch.cuda.synchronize()
    finally:
        set_option(b"tensor_core_backward", 1)
    out = {k: getattr(m, k).detach().cpu().numpy().copy() for k in ("theta", "theta_tgt", "adam_m", "adam_v")}
    out["metrics"] = metrics.detach().cpu().numpy().copy()
    if std:
        mean, var, count = m.ret_ms()
        out["ret_ms"] = np.concatenate([mean.numpy(), var.numpy()])
        out["ret_count"] = np.array([count])
    if cls == "QMixNetwork":
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

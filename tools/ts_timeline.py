"""Timeline of one IDQN update from the probes of a -DMARL_TC_TIMESTAMPS build (python codebase_b200/csrc/build.py --timestamps; run with
MARL_B200_SO=codebase_b200/csrc/libmarlb200_ts.so).  Prints, per kernel of the last update: first CTA start / last CTA end on the global timer
(relative to the update's first probe), and the median / max over CTAs of every probe slot relative to the CTA's own start (SM cycles)."""
import ctypes as C
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from codebase_b200 import _native as nat   # noqa: E402
from codebase_b200.lbf import TrajStore   # noqa: E402
import types   # noqa: E402

NAMES = {0: "tc_forward (target)", 1: "tc_dqn_fwd", 2: "tc_dh1", 3: "tc_dw", 4: "reduce_adam"}


def main():
    from codebase_b200.dqn.model import QNetwork

    B, T, D, A, N = 1024, 25, 15, 6, 2
    sp = lambda **k: types.SimpleNamespace(**k)
    cfg = sp(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=1.0, double_q=True, target_update_interval_or_tau=200, standardise_returns=False)
    m = QNetwork([sp(shape=(D,), n=None)] * N, [sp(n=A, shape=None)] * N, cfg, [128, 128], False, False, True, "cuda", max_batch=B, max_episode_length=T)
    cap = 10000
    rb = TrajStore(cap, N, T, D, m.device)
    g = torch.Generator(device="cuda").manual_seed(0)
    rb.obs.copy_(torch.randint(-1, 8, rb.obs.shape, device="cuda", generator=g).float())
    rb.act.copy_(torch.randint(0, A, rb.act.shape, device="cuda", generator=g).int())
    rb.rew.copy_(torch.rand(rb.rew.shape, device="cuda", generator=g))
    rb.filled.fill_(1)
    m.update_n(rb, B, cap, 1, 0, 64)
    torch.cuda.synchronize()
    buf = np.zeros((160, 32, 2), np.uint64)
    data = {}
    for k in NAMES:
        rc = nat.lib().marl_debug_timestamps(C.c_int32(k), buf.ctypes.data_as(C.POINTER(C.c_uint64)))
        if rc == 0 and buf[:, 0, 0].max() > 0:
            data[k] = buf.copy()
    t0 = min(int(d[:, 0, 0][d[:, 0, 0] > 0].min()) for d in data.values())
    last = max(int(d[:, :, 0].max()) for d in data.values())
    live = {k: d for k, d in data.items() if int(d[:, :, 0].max()) > last - 400_000}   # probes written by the last update only
    order = sorted(live, key=lambda k: int(live[k][:, 0, 0][live[k][:, 0, 0] > 0].min()))
    t0 = min(int(live[k][:, 0, 0][live[k][:, 0, 0] > 0].min()) for k in order)
    for k in order:
        d = live[k]
        ctas = d[:, 0, 0] > 0
        g0 = d[ctas, 0, 0].astype(np.int64) - t0
        ends = d[ctas][:, :, 0].max(axis=1).astype(np.int64) - t0
        print(f"== {NAMES[k]}: {int(ctas.sum())} CTAs; first start {g0.min() / 1e3:.1f} us, last start {g0.max() / 1e3:.1f}, first end {ends.min() / 1e3:.1f}, last end {ends.max() / 1e3:.1f} us")
        c = d[ctas][:, :, 1].astype(np.int64)
        gt = d[ctas][:, :, 0].astype(np.int64)
        rows = []
        for s in range(32):
            ok = gt[:, s] >= gt[:, 0]
            ok &= d[ctas][:, s, 0] > 0
            if ok.sum() < max(1, ctas.sum() // 2):
                continue
            rel = (c[ok, s] - c[ok, 0])
            rows.append(f"   slot {s:2d}: median {int(np.median(rel)):7d} cyc  max {int(rel.max()):7d}   (global: median +{np.median(gt[ok, s] - t0) / 1e3:.1f} us)")
        print("\n".join(rows))


if __name__ == "__main__":
    main()

"""GPU: destroying a learner handle releases every device buffer it owns, including the ones allocated on first use (tensor-core
intermediates, PPO buffers, the QMIX mixer, return statistics, the peer-exchange buffer).  Each case creates, uses and destroys a handle
20 times; this process's device memory, as NVML reports it, must not grow between the first cycle and the last."""
import ctypes as C
import os
import types

import numpy as np
import pytest
import torch

from tests.helpers import ac_batch, ac_model, random_store, space, traj_store

pytestmark = pytest.mark.gpu
N, D, A, T, B = 2, 15, 6, 25, 256
CYCLES = 20
SLACK = 1 << 20   # bytes; a leaked lazily allocated buffer set of any case below costs more than this over 19 cycles


def _process_bytes():
    """device memory of this process summed over the GPUs, or None when NVML cannot attribute memory to it (e.g. another PID namespace)"""
    import pynvml

    pynvml.nvmlInit()
    try:
        total, seen = 0, False
        for i in range(pynvml.nvmlDeviceGetCount()):
            for p in pynvml.nvmlDeviceGetComputeRunningProcesses(pynvml.nvmlDeviceGetHandleByIndex(i)):
                if p.pid == os.getpid():
                    if p.usedGpuMemory is None:
                        return None
                    total, seen = total + p.usedGpuMemory, True
        return total if seen else None
    finally:
        pynvml.nvmlShutdown()


def _dqn(cls="QNetwork", use_rnn=False, standardise=False, mixing=None):
    from codebase_b200.dqn import model as M

    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=1.0, double_q=True, target_update_interval_or_tau=200,
                                standardise_returns=standardise)
    args = ([space(shape=(D,))] * N, [space(n=A)] * N, cfg, [128, 128], False, use_rnn, True)
    if mixing is not None:
        args += (mixing,)
    return getattr(M, cls)(*args, "cuda", max_batch=B, max_episode_length=T)


def _ac(cls, centralised=False, standardise=False):
    hp = types.SimpleNamespace(lr=3e-4, gamma=0.99, grad_clip=0.5, n_steps=5, entropy_coef=0.01, value_loss_coef=0.5, target_update_interval_or_tau=200)
    return ac_model(hp, N, D, B, T, A, cls=cls, centralised=centralised, standardise=standardise)


def _peer_handle(m):
    buf = (C.c_ubyte * 64)()
    assert m._lib.marl_dqn_peer_handle(m._h, buf) == 0


# name -> (make the handle, use it); the data are made once, outside the cycles
CASES = {
    "idqn_tensor_core_update": (lambda: _dqn(), lambda m, d: m.update_from_store(d["replay"], d["idx"])),
    "vdn_standardise_returns": (lambda: _dqn("VDNetwork", standardise=True), lambda m, d: m.update_from_store(d["replay"], d["idx"])),
    "qmix": (lambda: _dqn("QMixNetwork", mixing=dict(embed_dim=32, hypernet_layers=2, hypernet_embed=64)),
             lambda m, d: m.update_from_store(d["replay"], d["idx"])),
    "idqn_rnn": (lambda: _dqn(use_rnn=True), lambda m, d: m.update_from_store(d["replay"], d["idx"])),
    "ppo_update": (lambda: _ac("PPONetwork"), lambda m, d: m.update_from_store(d["batch"], B, 1)),
    "maa2c_standardise_returns": (lambda: _ac("A2CNetwork", centralised=True, standardise=True), lambda m, d: m.update_from_store(d["batch"], B, 1)),
    "dqn_peer_handle": (lambda: _dqn(), lambda m, d: _peer_handle(m)),
}


@pytest.mark.parametrize("case", list(CASES))
def test_destroy_releases_every_buffer(case):
    make, use = CASES[case]
    rng = np.random.default_rng(7)
    dev = torch.device("cuda")
    data = dict(replay=traj_store(random_store(rng, 2 * B, N, T, D, coop=True), dev), batch=traj_store(ac_batch(rng, B, N, T, D), dev),
                idx=torch.as_tensor(rng.integers(0, 2 * B, size=B).astype(np.int32), device=dev))
    readings = []
    for c in range(CYCLES):
        m = make()
        use(m, data)
        torch.cuda.synchronize()
        m.close()
        del m
        if c in (0, CYCLES - 1):
            torch.cuda.empty_cache()
            readings.append(_process_bytes())
            if readings[-1] is None:
                pytest.skip("NVML does not report this process's device memory here (the process is not listed, e.g. a separate PID namespace)")
    first, last = readings
    assert last - first <= SLACK, f"{case}: this process holds {last - first} more bytes after {CYCLES} cycles than after the first"

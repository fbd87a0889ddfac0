"""GPU: the three-kernel wgmma training pipeline (tc_train.cu, option "tensor_core_backward") against the fused FP32 kernel and
the CPU oracle: gradients, loss, parameters after the update -- IDQN and VDN, ragged tiles, obs widths 15 / 27, several T."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

from oracle import learner_ref as lr

from tests.helpers import check_margin, redraw_on_near_tie, assert_grad_close

pytestmark = pytest.mark.gpu
A = 6


def _space(shape=None, n=None):
    return types.SimpleNamespace(shape=shape, n=n)


def _opt(name, on):
    from codebase_b200 import _native as nat

    nat.check(nat.lib().marl_set_option(name, C.c_int32(int(on))), "marl_set_option")


@pytest.fixture(autouse=True)
def _restore():
    yield
    _opt(b"tensor_core_backward", True)   # the library defaults
    _opt(b"tensor_core_forward", True)


def _store(rng, cap, N, T, D, coop):
    obs = rng.integers(-1, 12, size=(cap, N, T + 1, D)).astype(np.float32)
    act = rng.integers(0, A, size=(cap, N, T)).astype(np.int32)
    rew = (rng.random((cap, N, T)) < 0.2).astype(np.float32) * rng.random((cap, N, T)).astype(np.float32)
    if coop:
        rew[:] = rew[:, :1]
    length = rng.integers(1, T + 1, size=cap)
    done = np.zeros((cap, T + 1), np.uint8); filled = np.zeros((cap, T), np.uint8)
    for e in range(cap):
        filled[e, : length[e]] = 1
        done[e, length[e]] = rng.random() < 0.8
    return dict(obs=obs, act=act, rew=rew, done=done, filled=filled)


@pytest.mark.parametrize("mixer,N,D,T,B,sharing", [(0, 2, 15, 25, 64, False), (0, 2, 15, 25, 1024, False), (1, 2, 15, 25, 257, False),
                                                   (0, 4, 27, 25, 96, False), (0, 2, 15, 50, 100, True), (0, 3, 15, 7, 333, [0, 1, 0]), (1, 4, 27, 25, 48, False)])
@redraw_on_near_tie
def test_tc_backward_matches_ffma_and_oracle(mixer, N, D, T, B, sharing):
    from codebase_b200.dqn import model as M
    from codebase_b200.lbf import TrajStore

    rng = np.random.default_rng(B * 7 + T)
    hp = lr.DqnHP(mixer=mixer)
    cfg = types.SimpleNamespace(optimizer="Adam", lr=hp.lr, gamma=hp.gamma, grad_clip=hp.grad_clip, double_q=True, target_update_interval_or_tau=200, standardise_returns=False)
    m = (M.VDNetwork if mixer else M.QNetwork)([_space(shape=(D,))] * N, [_space(n=A)] * N, cfg, [128, 128], sharing, False, True, "cuda", max_batch=B, max_episode_length=T)
    # perturbations from the seeded numpy stream: an unseeded CUDA draw makes the case vary from run to run, and a near-tie in the
    # double-Q argmax (GPU and oracle outputs differ by ~1e-6) then flips one target -- a 2e-5 gradient difference that is not a bug
    noise = lambda s_: torch.as_tensor(s_ * rng.standard_normal(m.theta.numel()), dtype=torch.float32).to(m.theta.device).view_as(m.theta)
    m.theta.add_(noise(0.02)); m.hard_update(); m.theta.add_(noise(0.01)); m.params_changed()  # direct writes
    st = lr.DqnState(m.theta.cpu().clone(), m.theta_tgt.cpu().clone(), m.agent_net, D, A)
    s = _store(rng, 300, N, T, D, bool(mixer))
    idx = rng.integers(0, 300, size=B).astype(np.int32)
    batch = lr.batch_from_store(s, idx)
    check_margin(lr, st, batch, hp)   # near-tie in the double-Q argmax: re-drawn by the decorator
    st0 = lr.DqnState(st.theta.clone(), st.theta_tgt.clone(), st.agent_net, D, A)   # dqn_update steps st in place
    want = lr.dqn_update(st, batch, hp)
    ts = TrajStore(300, N, T, D, m.device)
    for k in ("obs", "act", "rew", "done", "filled"):
        getattr(ts, k).copy_(torch.as_tensor(s[k]))
    idx_d = torch.tensor(idx, device="cuda")
    n = m.n_params
    scale = max(1.0, float(np.abs(want["grad"].numpy()).max()))
    grads = {}
    # 0: fused FP32 kernel; 1: the tensor-core pipeline (the default; applied below)
    for tc in (0, 1):
        _opt(b"tensor_core_backward", tc)
        m.update_grads(ts, idx_d)
        torch.cuda.synchronize()
        g = m.grad.cpu().numpy()
        grads[tc] = g[:n] / g[n + 1]
        assert abs(g[n] / g[n + 1] - want["loss"]) <= 1e-5 * max(1.0, abs(want["loss"])), (tc, g[n] / g[n + 1], want["loss"])
        assert_grad_close(lr, st0, batch, hp, grads[tc], want["grad"].numpy(), what=f"kernel selection {tc}:")
    assert np.abs(grads[0] - grads[1]).max() / scale < 1e-5
    met = m.update_apply().cpu().numpy()  # applies the tensor-core gradients
    d = np.abs(m.theta.cpu().numpy() - st.theta.numpy())
    assert np.quantile(d, 0.999) < 1e-5 and abs(met[0] - want["loss"]) <= 1e-5 * max(1.0, abs(want["loss"]))

"""cfg.standardise_returns of the DQN family (marlbase/dqn/model.py:82-84,147-158; VDN 221-222,256-264): the oracle against outputs of the
reference classes stored under tests/golden, and the CUDA path (marl_dqn_standardise_returns) against the oracle."""
import copy
import os
import types

import numpy as np
import pytest
import torch

from oracle import learner_ref as lr
from tests.helpers import GOLDEN, STRIDE, assert_grad_close, check_margin, load_params, redraw_on_near_tie, reference_outputs, seeded_params

N, D, A, T = 2, 15, 6, 25


def _close(a, b, rtol=1e-5, atol=1e-5):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert np.allclose(a, b, rtol=rtol, atol=atol), float(np.abs(a - b).max())


def _space(shape=None, n=None):
    return types.SimpleNamespace(shape=shape, n=n)


def _store(rng, cap, coop):
    obs = rng.integers(-1, 8, size=(cap, N, T + 1, D)).astype(np.float32)
    act = rng.integers(0, A, size=(cap, N, T)).astype(np.int32)
    rew = 3.0 * (rng.random((cap, N, T)) < 0.3).astype(np.float32) * rng.random((cap, N, T)).astype(np.float32)
    if coop:
        rew[:] = rew[:, :1]
    length = rng.integers(1, T + 1, size=cap)
    done = np.zeros((cap, T + 1), np.uint8); filled = np.zeros((cap, T), np.uint8)
    for e in range(cap):
        filled[e, : length[e]] = 1
        done[e, length[e]] = rng.random() < 0.7
    return dict(obs=obs, act=act, rew=rew, done=done, filled=filled)


def _std_batches(mixer):
    rng = np.random.default_rng(8)
    for _ in range(3):
        s = _store(rng, 40, bool(mixer))
        yield lr.batch_from_store(s, rng.integers(0, 40, size=12).astype(np.int32))


@pytest.mark.parametrize("cls,mixer", [("QNetwork", 0), ("VDNetwork", 1)])
def test_oracle_matches_live_reference(cls, mixer):
    """three updates from seeded weights vs what the reference's classes computed for them (recorded from the live classes under tests/golden)"""
    g = reference_outputs("standardise_returns_reference")
    theta = seeded_params(lr, N, D, A, 3)
    st = lr.DqnState(theta.clone(), theta.clone(), [0, 1], D, A, ret_ms=lr.RunningMeanStdRef((1,) if mixer else (N,)))
    hp = lr.DqnHP(mixer=mixer)
    for u, b in enumerate(_std_batches(mixer)):
        _close(lr.dqn_update(st, b, hp)["loss"], g[f"{cls}_losses"][u])
    _close(st.ret_ms.mean.numpy(), g[f"{cls}_ret_mean"]); _close(st.ret_ms.var.numpy(), g[f"{cls}_ret_var"])
    assert np.quantile(np.abs(st.theta.numpy()[::STRIDE] - g[f"{cls}_theta"]), 0.999) < 1e-5


def make_reference_outputs(ref, ref_shim):
    """tests/golden/standardise_returns_reference.npz: the reference's QNetwork / VDNetwork with standardise_returns on the inputs above."""
    out = {}
    for cls, mixer in (("QNetwork", 0), ("VDNetwork", 1)):
        model = getattr(ref.dqn_model, cls)([ref_shim.Space(shape=(D,))] * N, [ref_shim.Space(n=A)] * N, ref_shim.dqn_cfg(standardise_returns=True), [128, 128], False, False, True, "cpu")
        load_params(model, lr, ("critic.independent", "target.independent"), seeded_params(lr, N, D, A, 3), N, D, A)
        out[f"{cls}_losses"] = np.array([model.update(ref.dqn_train.Batch(b["obss"], b["actions"], b["rewards"], b["dones"], b["filled"], None))["loss"]
                                         for b in _std_batches(mixer)], np.float64)
        out[f"{cls}_ret_mean"], out[f"{cls}_ret_var"] = model.ret_ms.mean.numpy(), model.ret_ms.var.numpy()
        out[f"{cls}_theta"] = lr.flat_from_state_dict(model.state_dict(), "critic.independent", N).numpy()[::STRIDE]
    np.savez_compressed(os.path.join(GOLDEN, "standardise_returns_reference.npz"), **out)


@pytest.mark.gpu
@pytest.mark.parametrize("mixer,B,sharing", [(0, 64, False), (0, 700, True), (1, 48, False), (1, 257, False)])
@redraw_on_near_tie
def test_device_matches_oracle(mixer, B, sharing):
    from codebase_b200.dqn import model as M
    from codebase_b200.lbf import TrajStore

    rng = np.random.default_rng(B)
    hp = lr.DqnHP(mixer=mixer, target_update_interval_or_tau=2)
    cfg = types.SimpleNamespace(optimizer="Adam", lr=hp.lr, gamma=hp.gamma, grad_clip=hp.grad_clip, double_q=True, target_update_interval_or_tau=2, standardise_returns=True)
    m = (M.VDNetwork if mixer else M.QNetwork)([_space(shape=(D,))] * N, [_space(n=A)] * N, cfg, [128, 128], sharing, False, True, "cuda", max_batch=B, max_episode_length=T)
    st = lr.DqnState(m.theta.cpu().clone(), m.theta_tgt.cpu().clone(), m.agent_net, D, A, ret_ms=lr.RunningMeanStdRef((1,) if mixer else (N,)))
    for u in range(3):
        s = _store(rng, 300, bool(mixer))
        idx = rng.integers(0, 300, size=B).astype(np.int32)
        batch = lr.batch_from_store(s, idx)
        check_margin(lr, st, batch, hp)   # a double-Q near-tie makes the comparison a coin toss: re-drawn by the decorator
        st0 = copy.deepcopy(st)           # dqn_update steps st in place; a ReLU kink is judged on the state before it
        want = lr.dqn_update(st, batch, hp)
        ts = TrajStore(300, N, T, D, m.device)
        for k in ("obs", "act", "rew", "done", "filled"):
            getattr(ts, k).copy_(torch.as_tensor(s[k]))
        m.update_grads(ts, torch.tensor(idx, device="cuda"))
        gr = m.grad.cpu().numpy(); n = m.n_params
        assert_grad_close(lr, st0, batch, hp, gr[:n] / gr[n + 1], want["grad"].numpy(), tol=2e-5, what=f"update {u}:")
        _close(m.update_apply().cpu().numpy()[0], want["loss"], rtol=2e-5, atol=2e-5)
        mean, var, count = m.ret_ms()
        ref_mean = st.ret_ms.mean.numpy() if st.ret_ms.mean.numel() > 1 else np.full(len(mean), float(st.ret_ms.mean))
        _close(mean.numpy(), ref_mean); _close(var.numpy(), st.ret_ms.var.numpy() if st.ret_ms.var.numel() > 1 else np.full(len(var), float(st.ret_ms.var)))
        assert abs(count - st.ret_ms.count) < 1e-6
        m.theta.copy_(st.theta); m.theta_tgt.copy_(st.theta_tgt); m.adam_m.copy_(st.m); m.adam_v.copy_(st.v)
        m.params_changed()

"""GPU: the fused IDQN / VDN learner kernels (through the C ABI) against golden vectors produced by the reference's own
classes and against the CPU oracle on seeded random batches.  Tolerance: 1e-5 (rtol and atol) on float learner tensors,
as BASELINE.json's north_star states."""
import os
import types

import numpy as np
import pytest
import torch

from oracle import learner_ref as lr
from oracle import policy_ref
from tests.helpers import NearTie, assert_grad_close, clipped as _clipped, close_scaled as _close_scaled, golden_stride, space as _space

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
N, D, A, T = 2, 15, 6, 25


def _close(a, b, rtol=1e-5, atol=1e-5):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert np.allclose(a, b, rtol=rtol, atol=atol), float(np.abs(a - b).max())


def _model(cls_name, sharing, hp, n_agents=N, max_batch=64):
    from codebase_b200.dqn import model as M

    cfg = types.SimpleNamespace(optimizer="Adam", lr=hp.lr, gamma=hp.gamma, grad_clip=hp.grad_clip, double_q=hp.double_q,
                                target_update_interval_or_tau=hp.target_update_interval_or_tau, standardise_returns=False)
    return getattr(M, cls_name)([_space(shape=(D,))] * n_agents, [_space(n=A)] * n_agents, cfg, [128, 128], sharing, False, True, "cuda",
                                max_batch=max_batch, max_episode_length=T)


def _store_to_device(store, device):
    from codebase_b200.lbf import TrajStore

    cap, n_agents = store["obs"].shape[0], store["obs"].shape[1]
    ts = TrajStore(cap, n_agents, T, D, device)
    for k in ("obs", "act", "rew", "done", "filled"):
        getattr(ts, k).copy_(torch.as_tensor(store[k]))
    return ts


def test_forward_matches_oracle():
    rng = np.random.default_rng(0)
    for sharing, E in ((False, 4096), (True, 1000), (False, 1), (False, 37)):
        m = _model("QNetwork", sharing, lr.DqnHP())
        theta = m.theta.cpu()
        obs = rng.integers(-1, 8, size=(E, N, D)).astype(np.float32)
        q = m.q_values(torch.tensor(obs, device="cuda")).cpu().numpy()
        want = torch.stack(lr.agents_forward(theta, m.agent_net, [torch.tensor(obs[:, i]) for i in range(N)], D, A), 1).numpy()
        _close(q, want)
        tq = m.q_values(torch.tensor(obs, device="cuda"), target=True).cpu().numpy()
        _close(tq, want)


@pytest.mark.parametrize("name", ["idqn_indep", "idqn_single_q_polyak_noclip", "idqn_shared", "vdn_indep"])
def test_update_matches_reference_golden(name):
    g = np.load(os.path.join(GOLD, f"{name}.npz"))
    hp = lr.DqnHP(lr=float(g["hp"][0]), gamma=float(g["hp"][1]), grad_clip=float(g["hp"][2]), double_q=bool(g["hp"][3]),
                  target_update_interval_or_tau=float(g["hp"][4]), mixer=int(g["mixer"]))
    m = _model("VDNetwork" if hp.mixer else "QNetwork", bool(int(g["n_nets"]) == 1), hp)
    assert m.n_params == g["theta0"].size
    m.theta.copy_(torch.tensor(g["theta0"])); m.params_changed(); m.hard_update()
    S = golden_stride(g)
    for u in range(len(g["losses"])):
        store = {k: g[f"u{u}_{k}"] for k in ("obs", "act", "rew", "done", "filled")}
        ts = _store_to_device(store, m.device)
        idx = torch.tensor(g[f"u{u}_idx"], dtype=torch.int32, device="cuda")
        if u == 0:
            m.update_grads(ts, idx)
            gr = m.grad.cpu().numpy()
            n = m.n_params
            _close((gr[:n] / gr[n + 1])[::S], g["grad0"])        # un-normalised sums / filled count == autograd gradient
            _close_scaled(_clipped(gr[:n] / gr[n + 1], hp.grad_clip)[::S], g["grad0_clipped"])   # element-wise, what Adam consumes
            _close(gr[n] / gr[n + 1], g["losses"][0])
            met = m.update_apply()
        else:
            met = m.update_from_store(ts, idx)
        _close(met[0].item(), g["losses"][u])
    # Adam state element-wise against the reference optimiser's exp_avg / exp_avg_sq: the quantile bound on theta cannot hide a defect here
    _close_scaled(m.adam_m.cpu().numpy()[::S], g["adam_m_final"])
    _close_scaled(m.adam_v.cpu().numpy()[::S], g["adam_v_final"], tol=2e-5)
    d = np.abs(m.theta.cpu().numpy()[::S] - g["theta_final"])
    assert np.quantile(d, 0.999) < 1e-5 and d.max() < 2 * hp.lr * len(g["losses"]) + 1e-6, (np.quantile(d, 0.999), d.max())
    dt = np.abs(m.theta_tgt.cpu().numpy()[::S] - g["target_final"])
    assert np.quantile(dt, 0.999) < 1e-5


TIE = 2e-5   # relative gap of the two best online Q-values under which the double-Q argmax may legitimately differ between two implementations


@pytest.mark.parametrize("mixer,sharing,B,n_agents", [(0, False, 64, 2), (0, False, 1024, 2), (1, False, 257, 2), (0, True, 100, 2), (0, [0, 1, 0], 33, 3), (1, False, 48, 4)])
def test_update_matches_oracle_on_random_batches(mixer, sharing, B, n_agents):
    """Three glued updates against the oracle.  A case whose oracle argmax margin is below TIE is re-drawn (new initialisation), at most four times:
    with a healthy margin every mismatch is a defect."""
    for attempt in range(5):
        torch.manual_seed(1000 * attempt + B)
        if _three_glued_updates(mixer, sharing, B, n_agents) == "ok":
            return
    pytest.fail("five initialisations in a row hit a double-Q near-tie: not plausible")


def _three_glued_updates(mixer, sharing, B, n_agents):
    rng = np.random.default_rng(B)
    hp = lr.DqnHP(mixer=mixer, target_update_interval_or_tau=2)
    m = _model("VDNetwork" if mixer else "QNetwork", sharing, hp, n_agents=n_agents, max_batch=B)
    st = lr.DqnState(m.theta.cpu().clone(), m.theta_tgt.cpu().clone(), m.agent_net, D, A)
    cap = 300
    for u in range(3):
        obs = rng.integers(-1, 8, size=(cap, n_agents, T + 1, D)).astype(np.float32)
        act = rng.integers(0, A, size=(cap, n_agents, T)).astype(np.int32)
        rew = (rng.random((cap, n_agents, T)) < 0.2).astype(np.float32) * rng.random((cap, n_agents, T)).astype(np.float32)
        if mixer:
            rew[:] = rew[:, :1]
        length = rng.integers(1, T + 1, size=cap)
        done = np.zeros((cap, T + 1), np.uint8); filled = np.zeros((cap, T), np.uint8)
        for e in range(cap):
            filled[e, : length[e]] = 1
            done[e, length[e]] = rng.random() < 0.7
        store = dict(obs=obs, act=act, rew=rew, done=done, filled=filled)
        idx = rng.integers(0, cap, size=B).astype(np.int32)
        batch = lr.batch_from_store(store, idx)
        if lr.double_q_margin(st, batch, hp) < TIE:
            return "near-tie"   # the comparison would be a coin toss on which target action is selected
        st_before = lr.DqnState(st.theta.clone(), st.theta_tgt.clone(), st.agent_net, D, A)
        want = lr.dqn_update(st, batch, hp)
        ts = _store_to_device(store, m.device)
        m.update_grads(ts, torch.tensor(idx, device="cuda"))
        gr = m.grad.cpu().numpy()
        try:   # ... or when a ReLU unit on its kink explains a mismatch (tests/helpers.py)
            assert_grad_close(lr, st_before, batch, hp, gr[:m.n_params] / gr[m.n_params + 1], want["grad"].numpy())
        except NearTie:
            return "near-tie"
        _close_scaled(_clipped(gr[:m.n_params] / gr[m.n_params + 1], hp.grad_clip), want["grad_clipped"].numpy())
        met = m.update_apply().cpu().numpy()
        _close(met[0], want["loss"]); _close(met[1], want["grad_norm"], rtol=1e-4)
        _close_scaled(m.adam_m.cpu().numpy(), st.m.numpy()); _close_scaled(m.adam_v.cpu().numpy(), st.v.numpy(), tol=2e-5)
        d = np.abs(m.theta.cpu().numpy() - st.theta.numpy())
        assert np.quantile(d, 0.999) < 1e-5 and d.max() < 2 * hp.lr * (u + 1) + 1e-6
        # keep the two trajectories glued so that later steps compare like for like
        m.theta.copy_(st.theta); m.theta_tgt.copy_(st.theta_tgt); m.adam_m.copy_(st.m); m.adam_v.copy_(st.v)
        m.params_changed()  # direct writes: cached derived data (packed target image) must be rebuilt
    assert m.updates == 3
    return "ok"


def test_reference_style_update_call_and_state_dict_roundtrip():
    """model.update(Batch) with the reference's Batch layout and reference-compatible checkpoint keys."""
    from collections import namedtuple

    Batch = namedtuple("Batch", ["obss", "actions", "rewards", "dones", "filled", "action_mask"])
    rng = np.random.default_rng(2)
    hp = lr.DqnHP()
    m = _model("QNetwork", False, hp)
    st = lr.DqnState(m.theta.cpu().clone(), m.theta_tgt.cpu().clone(), m.agent_net, D, A)
    B = 32
    b = dict(obss=torch.tensor(rng.standard_normal((N, T + 1, B, D)), dtype=torch.float32), actions=torch.tensor(rng.integers(0, A, (N, T, B))),
             rewards=torch.tensor(rng.random((N, T, B)), dtype=torch.float32), dones=torch.tensor(rng.random((T + 1, B)) < 0.05, dtype=torch.float32),
             filled=torch.tensor(rng.random((T, B)) < 0.9, dtype=torch.float32))
    want = lr.dqn_update(st, b, hp)
    got = m.update(Batch(*[b[k].cuda() for k in ("obss", "actions", "rewards", "dones", "filled")], None))
    _close(got["loss"], want["loss"])
    sd = m.state_dict()
    assert list(sd)[:2] == ["critic.independent.0.network.0.weight", "critic.independent.0.network.0.bias"]
    assert sd["critic.independent.1.network.4.weight"].shape == (A, 128) and "target.independent.0.network.2.bias" in sd
    m2 = _model("QNetwork", False, hp)
    m2.load_state_dict(sd)
    assert torch.equal(m2.theta, m.theta) and torch.equal(m2.theta_tgt, m.theta_tgt)


def test_replay_sampling_stream():
    from codebase_b200 import _native as nat
    import ctypes as C

    idx = torch.zeros(1000, dtype=torch.int32, device="cuda")
    for upd, n_valid in ((0, 10), (7, 65536), (2**33 + 5, 999)):
        nat.check(nat.lib().marl_replay_sample(C.c_uint64(99), C.c_uint64(upd), C.c_int32(1000), C.c_int32(n_valid), nat.ptr(idx), nat.stream_ptr()), "sample")
        assert np.array_equal(idx.cpu().numpy(), policy_ref.replay_sample(99, upd, 1000, n_valid))

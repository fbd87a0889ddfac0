"""Hidden widths other than 128 (`layers: [H, H]`, 1 <= H <= 128) on the GPU: the FP32 kernels with zero-padded 128-wide tiles over compact
parameters, against the oracle (oracle/learner_ref.py, oracle/qmix_ref.py with tests/hidden_width_ref.py's width-H networks) and the reference's fixture (tests/test_hidden_width.py)."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

from oracle import learner_ref as lr
from tests import hidden_width_ref as hr
from tests import test_hidden_width as hw
from tests.helpers import STRIDE, ac_batch, ac_oracle_batch, random_store, reference_outputs, space, traj_store

pytestmark = pytest.mark.gpu

A = 6


def _opt(name, on):
    from codebase_b200 import _native as nat

    nat.check(nat.lib().marl_set_option(name, C.c_int32(int(on))), "marl_set_option")


def _dqn_cfg(tu=200, clip=1.0, standardise=False):
    return types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=clip, double_q=True, target_update_interval_or_tau=tu,
                                 standardise_returns=standardise)


def _ac_cfg(clip=0.0, standardise=False, optimizer="Adam"):
    return types.SimpleNamespace(optimizer=optimizer, lr=3e-4, gamma=0.99, grad_clip=clip, n_steps=5, entropy_coef=0.001, value_loss_coef=0.5,
                                 target_update_interval_or_tau=2, standardise_returns=standardise, num_epochs=hw.EPOCHS, ppo_clip=0.2)


def _net(H, sharing=False, rnn=False, central=False):
    return types.SimpleNamespace(layers=[H, H], parameter_sharing=sharing, use_rnn=rnn, use_orthogonal_init=True, centralised=central)


def dqn_model(mixer, N, D, H, sharing=False, rnn=False, cfg=None, B=8, T=6):
    from codebase_b200.dqn import model as M

    cls = {0: M.QNetwork, 1: M.VDNetwork}.get(mixer)
    obs, act = [space(shape=(D,))] * N, [space(n=A)] * N
    if mixer == 2:
        return M.QMixNetwork(obs, act, cfg or _dqn_cfg(), [H, H], sharing, rnn, True, hw.MIXING, "cuda", max_batch=B, max_episode_length=T)
    return cls(obs, act, cfg or _dqn_cfg(), [H, H], sharing, rnn, True, "cuda", max_batch=B, max_episode_length=T)


def _close(a, b, tol=1e-5):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert np.abs(a - b).max() <= tol * max(1.0, float(np.abs(b).max())), float(np.abs(a - b).max())


# ---- forward parity -----------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [1, 37, 64, 100])
@pytest.mark.parametrize("E,sharing", [(3, False), (300, True), (700, False)])
def test_dqn_q_values(H, E, sharing):
    """q_values and the target network's on ragged (3) and multi-tile (300, 700 rows per agent) row counts"""
    N, D = 3, 11
    m = dqn_model(0, N, D, H, sharing)
    m.theta_tgt.copy_(m.theta * 0.5)
    obs = torch.randn(E, N, D, device="cuda")
    xs = [obs[:, i].cpu() for i in range(N)]
    for target, flat in ((False, m.theta), (True, m.theta_tgt)):
        assert hr.width_of(flat, m.agent_net, D, A) == H
        want = torch.stack(hr.agents_forward(flat.cpu(), m.agent_net, xs, D, A), 1)
        _close(m.q_values(obs, target=target).cpu(), want)
    m.close()


@pytest.mark.parametrize("H", [1, 37, 64, 100])
def test_ac_logits_and_values(H):
    from codebase_b200.ac import model as M

    N, D, E = 2, 40, 130   # 40 features: the KP = 64 tile
    m = M.A2CNetwork([space(shape=(D,))] * N, [space(n=A)] * N, _ac_cfg(), _net(H), _net(101 - H, central=True), "cuda", max_envs=8, max_episode_length=5)
    obs = torch.randn(E, N, D, device="cuda")
    xs = [obs[:, i].cpu() for i in range(N)]
    assert hr.width_of(m.actor_params, m.actor_net, D, A) == H and hr.width_of(m.critic_params, m.critic_net, N * D, 1) == 101 - H
    _close(m.logits(obs).cpu(), torch.stack(hr.agents_forward(m.actor_params.cpu(), m.actor_net, xs, D, A), 1))
    joint = obs.reshape(E, N * D).cpu()
    want_v = torch.cat(hr.agents_forward(m.critic_params.cpu(), m.critic_net, [joint] * N, N * D, 1), -1)
    _close(m.values(obs).cpu(), want_v)
    _close(m.values(obs, target=True).cpu(), want_v)
    m.close()


# ---- the fixture cases through the GPU path -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(hw.DQN_CASES))
def test_dqn_family_matches_reference(name):
    mixer, rnn, H, sharing, tu, seed = hw.DQN_CASES[name]
    g = reference_outputs("hidden_width_reference")
    st, hp, store, idx = hw.dqn_setup(name)
    m = dqn_model(mixer, hw.N, hw.DQN_D, H, sharing, rnn, _dqn_cfg(tu=tu), B=hw.DQN_B, T=hw.DQN_T)
    m.theta.copy_(st.theta); m.theta_tgt.copy_(st.theta_tgt); m.params_changed()
    if mixer == 2:
        m.mix.copy_(st.mix); m.mix_tgt.copy_(st.mix_tgt)
    ts = traj_store(store, m.device)
    for u in range(hw.UPDATES):
        loss = float(m.update_from_store(ts, torch.tensor(idx[u], device="cuda"))[0])
        want = float(g[f"{name}_loss"][u])
        assert abs(loss - want) <= 1e-5 * max(1.0, abs(want)), (u, loss, want)
    for mine, key in ((m.theta, "theta"), (m.theta_tgt, "theta_tgt")) + (((m.mix, "mix"),) if mixer == 2 else ()):
        d = np.abs(mine.cpu().numpy()[::STRIDE] - g[f"{name}_{key}"])
        assert np.quantile(d, 0.999) < 1e-5, (key, d.max())
    m.close()


@pytest.mark.parametrize("name", list(hw.AC_CASES))
def test_ac_family_matches_reference(name):
    from codebase_b200.ac import model as M

    cls, ah, arnn, ch, crnn, central, sharing, clip, seed = hw.AC_CASES[name]
    g = reference_outputs("hidden_width_reference")
    st, hp, batches = hw.ac_setup(name)
    m = getattr(M, cls)([space(shape=(hw.AC_D,))] * hw.N, [space(n=A)] * hw.N, _ac_cfg(clip=clip), _net(ah, sharing, arnn), _net(ch, sharing, crnn, central),
                        "cuda", max_envs=hw.AC_P, max_episode_length=hw.AC_T)
    m.theta.copy_(torch.cat([st.actor, st.critic])); m.theta_tgt.copy_(st.target)
    metrics = []
    for step, s in zip(hw.AC_STEPS, batches):
        d = m.metrics_dict(m.update_from_store(traj_store(s, m.device), hw.AC_P, step))
        metrics.append([d[k] for k in ("loss", "actor_loss", "value_loss", "entropy")])
    assert np.allclose(metrics, g[f"{name}_metrics"], rtol=2e-5, atol=2e-5), (metrics, g[f"{name}_metrics"])
    for mine, key in ((m.actor_params, "actor"), (m.critic_params, "critic"), (m.theta_tgt, "target")):
        d = np.abs(mine.cpu().numpy()[::STRIDE] - g[f"{name}_{key}"])
        assert np.quantile(d, 0.999) < 1e-5, (key, d.max())
    m.close()


# ---- update chains against the oracle -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mixer,H,sharing,tu,clip,rnn", [(0, 37, False, 0.05, 1.0, False), (1, 100, True, 2, 0.0, False), (2, 1, False, 2, 1.0, False),
                                                          (0, 64, True, 0.05, 1.0, True), (1, 64, False, 200, 1.0, True)])
def test_dqn_chain(mixer, H, sharing, tu, clip, rnn):
    """three updates in a row, never re-synchronised with the oracle: clipped and unclipped, Polyak and hard target updates"""
    from oracle import qmix_ref as qr

    N, D, B, T, cap = 2, 9, 16, 12, 24
    torch.manual_seed(5 + H)
    m = dqn_model(mixer, N, D, H, sharing, rnn, _dqn_cfg(tu=tu, clip=clip), B=B, T=T)
    theta = m.theta.cpu().clone()
    if mixer == 2:
        st = qr.QmixState(theta.clone(), theta.clone(), m.mix.cpu().clone(), m.mix_tgt.cpu().clone(), m.agent_net, D, A, hw.MIXING["embed_dim"], hw.MIXING["hypernet_embed"])
    else:
        st = lr.DqnState(theta.clone(), theta.clone(), m.agent_net, D, A)
    hp = lr.DqnHP(grad_clip=clip, target_update_interval_or_tau=tu, mixer=mixer)
    rng = np.random.default_rng(H)
    store = random_store(rng, cap, N, T, D, coop=mixer != 0)
    ts = traj_store(store, m.device)
    for u in range(3):
        idx = rng.integers(0, cap, size=B).astype(np.int32)
        b = lr.batch_from_store(store, idx)
        with hr.networks([(D, A)] if rnn else []):
            want = qr.qmix_update(st, b, hp) if mixer == 2 else lr.dqn_update(st, b, hp)
        got = float(m.update_from_store(ts, torch.tensor(idx, device="cuda"))[0])
        assert abs(got - want["loss"]) <= 2e-5 * max(1.0, abs(want["loss"])), (u, got, want["loss"])
    for mine, ref in ((m.theta, st.theta), (m.theta_tgt, st.theta_tgt)):
        d = np.abs(mine.cpu().numpy() - ref.numpy())
        assert np.quantile(d, 0.999) < 1e-5, d.max()
    m.close()


@pytest.mark.parametrize("cls,ah,arnn,ch,crnn,central,sharing,clip,standardise", [
    ("A2CNetwork", 100, False, 1, False, False, False, 0.5, False),     # IA2C
    ("PPONetwork", 37, False, 64, False, False, True, 0.5, True),       # IPPO, standardise_returns
    ("A2CNetwork", 64, False, 37, False, True, False, 0.0, False),      # MAA2C
    ("PPONetwork", 64, True, 64, True, True, True, 0.5, False),         # MAPPO, both parts recurrent
])
def test_ac_chain(cls, ah, arnn, ch, crnn, central, sharing, clip, standardise):
    """three updates in a row (PPO: each of EPOCHS optimiser steps), never re-synchronised with the oracle"""
    from codebase_b200.ac import model as M

    N, D, P, T = 2, 9, 8, 12
    torch.manual_seed(ah + ch)
    m = getattr(M, cls)([space(shape=(D,))] * N, [space(n=A)] * N, _ac_cfg(clip=clip, standardise=standardise), _net(ah, sharing, arnn),
                        _net(ch, sharing, crnn, central), "cuda", max_envs=P, max_episode_length=T)
    nets = m.actor_net
    st = lr.A2CState(m.actor_params.cpu().clone(), m.critic_params.cpu().clone(), m.theta_tgt.cpu().clone(), nets, m.critic_net, D, A, centralised=central,
                     ret_ms=lr.RunningMeanStdRef((N,)) if standardise else None)
    hp = lr.A2CHP(grad_clip=clip, target_update_interval_or_tau=2)
    with hr.networks([(D, A)] * arnn + [(N * D if central else D, 1)] * crnn):
        rng = np.random.default_rng(ah * 7 + ch)
        for step in range(3):
            s = ac_batch(rng, P, N, T, D, A)
            want = lr.ppo_update(st, ac_oracle_batch(s), hp, step, hw.EPOCHS, 0.2) if cls == "PPONetwork" else lr.a2c_update(st, ac_oracle_batch(s), hp, step)
            got = m.metrics_dict(m.update_from_store(traj_store(s, m.device), P, step))
            assert abs(got["loss"] - want["loss"]) <= 5e-5 * max(1.0, abs(want["loss"])), (step, got["loss"], want["loss"])
    for mine, ref in ((m.actor_params, st.actor), (m.critic_params, st.critic), (m.theta_tgt, st.target)):
        d = np.abs(mine.cpu().numpy() - ref.numpy())
        assert np.quantile(d, 0.999) < 1e-5, d.max()
    m.close()


def test_dqn_update_n_sgd_matches_separate_updates():
    """marl_dqn_update_n (on-device replay sampling, fused tail) with a non-Adam optimiser at H = 37 gives what the same updates give one by one"""
    N, D, B, T, cap, K = 2, 9, 16, 12, 24, 4
    cfg = _dqn_cfg(tu=0.05)
    cfg.optimizer = "SGD"
    torch.manual_seed(3)
    a = dqn_model(0, N, D, 37, False, False, cfg, B=B, T=T)
    b = dqn_model(0, N, D, 37, False, False, cfg, B=B, T=T)
    b.theta.copy_(a.theta); b.theta_tgt.copy_(a.theta_tgt); b.params_changed()
    store = random_store(np.random.default_rng(9), cap, N, T, D, coop=False)
    ts = traj_store(store, a.device)
    a.update_n(ts, B, cap, 1234, 0, K)
    from codebase_b200 import _native as nat

    idx = torch.empty(B, dtype=torch.int32, device="cuda")
    for u in range(K):
        nat.check(nat.lib().marl_replay_sample(C.c_uint64(1234), C.c_uint64(u), C.c_int32(B), C.c_int32(cap), nat.ptr(idx), nat.stream_ptr()), "marl_replay_sample")
        b.update_from_store(ts, idx)
    torch.cuda.synchronize()
    assert torch.equal(a.theta, b.theta) and torch.equal(a.theta_tgt, b.theta_tgt)
    a.close(); b.close()


# ---- recurrent forward carrying the hidden state ------------------------------------------------------------------------------------------------
def test_gru_act_steps_carry_h_of_width_64():
    from codebase_b200.ac import model as AM

    N, D, E, S, H = 3, 9, 37, 5, 64
    m = dqn_model(0, N, D, H, False, True)
    assert m.init_hiddens(E)[0].shape == (1, E, H)
    obs = torch.randn(S, E, N, D)
    want_q, want_h = hr.act_steps(m.theta.cpu(), m.agent_net, obs, D, A)
    h = None
    for s in range(S):
        q, h_new = m.q_values(obs[s].cuda(), h=h)
        _close(q.cpu(), want_q[s]); _close(h_new.cpu(), want_h[s])
        h = h_new.clone()
    m.close()
    am = AM.A2CNetwork([space(shape=(D,))] * N, [space(n=A)] * N, _ac_cfg(), _net(H, rnn=True), _net(37, rnn=True), "cuda", max_envs=4, max_episode_length=5)
    assert am.init_actor_hiddens(E)[0].shape == (1, E, H) and am.init_critic_hiddens(E)[0].shape == (1, E, 37)
    want_q, want_h = hr.act_steps(am.actor_params.cpu(), am.actor_net, obs, D, A)
    lg, ho = am.logits(obs[0].cuda())
    _close(lg.cpu(), want_q[0]); _close(ho.cpu(), want_h[0])
    want_v, want_hc = hr.act_steps(am.critic_params.cpu(), am.critic_net, obs, D, 1)
    v, hc = am.values(obs[0].cuda())
    _close(v.cpu(), want_v[0][..., 0]); _close(hc.cpu(), want_hc[0])
    am.close()


# ---- the tensor-core options do not reach a narrower network -----------------------------------------------------------------------------------
@pytest.mark.parametrize("mixer", [0, 2])
def test_tensor_core_options_do_not_change_h64(mixer):
    """at H = 64 the handle has no packed image: tensor_core_forward / _backward on and off give bit-identical results"""
    N, D, B, T, cap = 2, 9, 16, 12, 24
    store = random_store(np.random.default_rng(4), cap, N, T, D, coop=mixer != 0)
    results = []
    try:
        for on in (True, False):
            _opt(b"tensor_core_forward", on); _opt(b"tensor_core_backward", on)
            torch.manual_seed(8)
            m = dqn_model(mixer, N, D, 64, False, False, B=B, T=T)
            ts = traj_store(store, m.device)
            rng = np.random.default_rng(1)
            for _ in range(3):
                m.update_from_store(ts, torch.tensor(rng.integers(0, cap, size=B).astype(np.int32), device="cuda"))
            q = m.q_values(torch.randn(50, N, D, generator=torch.Generator().manual_seed(2)).cuda())
            results.append((m.theta.clone(), m.theta_tgt.clone(), q.clone()))
            m.close()
    finally:
        _opt(b"tensor_core_forward", True); _opt(b"tensor_core_backward", True)
    for x, y in zip(*results):
        assert torch.equal(x, y)


# ---- the drivers end to end ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alg,env,extra", [
    ("idqn", "lbforaging:Foraging-8x8-2p-3f-v3", ["algorithm.model.layers=[64,64]", "algorithm.batch_size=128", "algorithm.buffer_size=4096"]),
    ("qmix", "lbforaging:Foraging-8x8-2p-3f-v3", ["algorithm.model.layers=[37,37]", "algorithm.batch_size=128", "algorithm.buffer_size=4096"]),
    ("ippo", "rware:rware-tiny-2ag-v2", ["algorithm.model.actor.layers=[64,64]", "algorithm.model.critic.layers=[32,32]"]),
])
def test_drivers_and_checkpoint_eval(tmp_path, monkeypatch, alg, env, extra):
    import pandas as pd

    from codebase_b200 import eval as ev
    from codebase_b200 import run

    monkeypatch.chdir(tmp_path)
    out = f"{tmp_path}/out"
    T = 25 if alg != "ippo" else 100
    run.main([f"+algorithm={alg}", f"env.name={env}", f"env.time_limit={T}", "env.parallel_envs=64", "seed=0", "algorithm.total_steps=20000",
              "algorithm.eval_interval=10000", "algorithm.save_interval=10000", f"run_dir={out}"] + extra)
    df = pd.read_csv(f"{out}/results.csv")
    assert len(df) >= 1 and np.isfinite(df["loss"]).all()
    monkeypatch.chdir(tmp_path)
    res = ev.main([f"path={out}", "episodes=16", "seed=3"])
    assert res["episodes"] == 16 and np.isfinite(res["mean_episode_returns"])

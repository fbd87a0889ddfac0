"""IPPO (marlbase/ac/model.py PPONetwork, 249-352): the oracle restatement against outputs of the reference classes stored under tests/golden,
and the CUDA path (marl_ppo_update through ac.model.PPONetwork) against the oracle on random on-policy batches; driver test."""
import copy
import os

import numpy as np
import pytest
import torch

from oracle import learner_ref as lr
from tests.helpers import GOLDEN, STRIDE, ac_batch, ac_model, ac_oracle_batch, load_params, reference_outputs, seeded_params, traj_store

N, D, A, T = 2, 15, 6, 25


def _close(a, b, rtol=1e-5, atol=1e-5):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert np.allclose(a, b, rtol=rtol, atol=atol), float(np.abs(a - b).max())


METRICS = ("loss", "actor_loss", "value_loss", "entropy")
# (fixture key, class, seed, batch seed, envs P, steps, epochs, grad_clip, parameter sharing, centralised critic, standardise_returns)
REF_CASES = {
    "std_a2c": ("A2CNetwork", 9, 3, 10, (0, 2, 3), 3, False, False, False, True),
    "std_ppo": ("PPONetwork", 9, 3, 10, (0, 2, 3), 3, False, False, False, True),
    "cent_a2c": ("A2CNetwork", 4, 5, 10, (0, 2, 3), 3, False, False, True, False),
    "cent_ppo": ("PPONetwork", 4, 5, 10, (0, 2, 3), 3, False, False, True, False),
    "ppo_indep": ("PPONetwork", 5, 11, 12, (0, 2, 5), 4, False, False, False, False),
    "ppo_shared_clip": ("PPONetwork", 5, 11, 12, (0, 2, 5), 4, 0.5, True, False, False),
}


def _ref_state(key):
    """The oracle state a case starts from: seeded weights (actor, critic; the target critic is a copy of the critic)."""
    cls, seed, _, _, _, _, clip, sharing, centralised, std = REF_CASES[key]
    n_nets, nets = (1, [0, 0]) if sharing else (N, [0, 1])
    actor, critic = seeded_params(lr, n_nets, D, A, seed), seeded_params(lr, n_nets, N * D if centralised else D, 1, seed + 1)
    return lr.A2CState(actor, critic.clone(), critic.clone(), nets, nets, D, A, centralised=centralised, ret_ms=lr.RunningMeanStdRef((N,)) if std else None)


def _run_oracle(key):
    cls, _, bseed, P, steps, epochs, clip, _, _, _ = REF_CASES[key]
    st = _ref_state(key)
    hp = lr.A2CHP(grad_clip=float(clip or 0.0), target_update_interval_or_tau=2)
    rng = np.random.default_rng(bseed)
    metrics = []
    for step in steps:
        b = ac_oracle_batch(ac_batch(rng, P, N, T, D))
        got = lr.ppo_update(st, b, hp, step, epochs, 0.2) if cls == "PPONetwork" else lr.a2c_update(st, b, hp, step)
        metrics.append([got[k] for k in METRICS])
    return st, metrics


def _check_reference_case(key):
    """oracle.learner_ref from the case's seeded weights and batches vs what the reference's A2CNetwork / PPONetwork computed for them (recorded
    from the live classes under tests/golden): losses, running return statistics, actor / critic / target parameters"""
    g = reference_outputs("ac_reference")
    st, metrics = _run_oracle(key)
    _close(metrics, g[f"{key}_metrics"])
    if REF_CASES[key][-1]:
        _close(st.ret_ms.mean.numpy(), g[f"{key}_ret_mean"]); _close(st.ret_ms.var.numpy(), g[f"{key}_ret_var"])
        assert abs(st.ret_ms.count - float(g[f"{key}_ret_count"])) < 1e-9
    for mine, name in ((st.actor, "actor"), (st.critic, "critic"), (st.target, "target")):
        d = np.abs(mine.numpy()[::STRIDE] - g[f"{key}_{name}"])
        assert np.quantile(d, 0.999) < 1e-5, (name, d.max())


@pytest.mark.parametrize("cls", ["A2CNetwork", "PPONetwork"])
def test_oracle_standardise_returns_matches_live_reference(cls):
    """cfg.standardise_returns=True: RunningMeanStd over the n-step returns (ac/model.py:195-204, 272-281)"""
    _check_reference_case("std_a2c" if cls == "A2CNetwork" else "std_ppo")


@pytest.mark.parametrize("cls", ["A2CNetwork", "PPONetwork"])
def test_oracle_centralised_critic_matches_live_reference(cls):
    """critic.centralised=True (MAA2C / MAPPO, ac/model.py:62-65,156-157)"""
    _check_reference_case("cent_a2c" if cls == "A2CNetwork" else "cent_ppo")


@pytest.mark.parametrize("sharing,clip", [(False, False), (True, 0.5)])
def test_oracle_ppo_matches_live_reference(sharing, clip):
    """three PPO updates (4 epochs each) of the reference's PPONetwork, without and with parameter sharing and gradient clipping"""
    _check_reference_case("ppo_shared_clip" if sharing else "ppo_indep")


def make_reference_outputs(ref, ref_shim):
    """tests/golden/ac_reference.npz: the reference's A2CNetwork / PPONetwork run on REF_CASES."""
    from collections import namedtuple

    Batch = namedtuple("Batch", ["obss", "actions", "rewards", "dones", "filled", "action_masks"])
    out = {}
    for key, (cls, _, bseed, P, steps, epochs, clip, sharing, centralised, std) in REF_CASES.items():
        st = _ref_state(key)
        cfg = ref_shim.a2c_cfg(grad_clip=clip, num_epochs=epochs, ppo_clip=0.2, target_update_interval_or_tau=2, standardise_returns=std)
        model = getattr(ref.ac_model, cls)([ref_shim.Space(shape=(D,))] * N, [ref_shim.Space(n=A)] * N, cfg, ref_shim.net_cfg(parameter_sharing=sharing),
                                           ref_shim.net_cfg(parameter_sharing=sharing, centralised=centralised), "cpu")
        kind, n_nets = ("networks", 1) if sharing else ("independent", N)
        load_params(model, lr, (f"actor.{kind}",), st.actor, n_nets, D, A)
        load_params(model, lr, (f"critic.{kind}", f"target_critic.{kind}"), st.critic, n_nets, N * D if centralised else D, 1)
        rng = np.random.default_rng(bseed)
        metrics = []
        for step in steps:
            b = ac_oracle_batch(ac_batch(rng, P, N, T, D))
            want = model.update(Batch(b["obss"], b["actions"], b["rewards"], b["dones"].bool(), b["filled"], None), step)
            metrics.append([float(want[k]) for k in METRICS])
        out[f"{key}_metrics"] = np.array(metrics, np.float64)
        if std:
            out[f"{key}_ret_mean"], out[f"{key}_ret_var"] = model.ret_ms.mean.numpy(), model.ret_ms.var.numpy()
            out[f"{key}_ret_count"] = np.float64(model.ret_ms.count)
        sd = model.state_dict()
        for name, prefix in (("actor", f"actor.{kind}"), ("critic", f"critic.{kind}"), ("target", f"target_critic.{kind}")):
            out[f"{key}_{name}"] = lr.flat_from_state_dict(sd, prefix, n_nets).numpy()[::STRIDE]
    np.savez_compressed(os.path.join(GOLDEN, "ac_reference.npz"), **out)


def test_oracle_ppo_first_epoch_is_a2c_with_unit_ratio():
    """epoch 0: ratio == 1 exactly, inside the clip range -> the surrogate's gradient is the policy gradient of A2C"""
    rng = np.random.default_rng(2)
    theta_a, theta_c = lr.init_flat(N, D, A), lr.init_flat(N, D, 1)
    b = ac_oracle_batch(ac_batch(rng, 8, N, T, D))
    st1 = lr.A2CState(theta_a.clone(), theta_c.clone(), theta_c.clone(), [0, 1], [0, 1], D, A)
    st2 = lr.A2CState(theta_a.clone(), theta_c.clone(), theta_c.clone(), [0, 1], [0, 1], D, A)
    g_ppo = lr.ppo_update(st1, b, lr.A2CHP(), 0, 1, 0.2)["grad"]
    g_a2c = lr.a2c_update(st2, b, lr.A2CHP(), 0)["grad"]
    _close(g_ppo["actor"].numpy(), g_a2c["actor"].numpy()); _close(g_ppo["critic"].numpy(), g_a2c["critic"].numpy())


def test_oracle_per_epoch_outputs_and_kink_risk():
    """ppo_update's per-epoch outputs keep `grad` as the first epoch's raw gradient; a2c_kink_risk is 0 where no hidden unit sits within 2e-6 of
    its kink, and positive once one unit's bias puts it 1e-7 from its kink on one row"""
    rng = np.random.default_rng(4)
    theta_a, theta_c = lr.init_flat(N, D, A, generator=torch.Generator().manual_seed(1)), lr.init_flat(N, D, 1, generator=torch.Generator().manual_seed(2))
    b = ac_oracle_batch(ac_batch(rng, 4, N, 6, D))
    st = lr.A2CState(theta_a.clone(), theta_c.clone(), theta_c.clone(), [0, 1], [0, 1], D, A)
    res = lr.ppo_update(st, b, lr.A2CHP(lr=3e-3), 0, 3, 0.2)
    assert len(res["grads"]) == len(res["grad_norms"]) == len(res["clip_frac"]) == len(res["clip_margin"]) == 3
    for k in ("actor", "critic"):
        assert torch.equal(res["grads"][0][k], res["grad"][k])
    assert res["grad_norms"][0] == pytest.approx(float(torch.cat([res["grad"]["actor"], res["grad"]["critic"]]).norm()), rel=1e-6)
    st = lr.A2CState(theta_a.clone(), theta_c.clone(), theta_c.clone(), [0, 1], [0, 1], D, A)
    assert lr.a2c_kink_risk(st, b, lr.A2CHP()) == 0.0
    w1, b1 = lr.split_net(st.actor, D, A)[:2]        # views into agent 0's actor network
    x = b["obss"][0, 0, :D]                          # step 0 of every episode is filled
    b1[7] = 1e-7 - float(w1[7] @ x)
    assert lr.a2c_kink_risk(st, b, lr.A2CHP()) > 0.0


def test_oracle_ppo_kink_risk():
    """ppo_kink_risk judges an epoch's loss at the parameters that epoch started from: 0 where no hidden unit sits within 2e-6 of its kink, positive
    once one actor unit is 1e-7 from its kink on a filled row (an all-zero observation row, so that the unit's pre-activation is its bias exactly)"""
    rng = np.random.default_rng(4)
    theta_a, theta_c = lr.init_flat(N, D, A, generator=torch.Generator().manual_seed(1)), lr.init_flat(N, D, 1, generator=torch.Generator().manual_seed(2))
    b = ac_oracle_batch(ac_batch(rng, 4, N, 6, D))
    b["obss"][0, 0, :D] = 0.0                        # step 0 of every episode is filled
    hp = lr.A2CHP(lr=3e-3)
    st = lr.A2CState(theta_a.clone(), theta_c.clone(), theta_c.clone(), [0, 1], [0, 1], D, A)
    st0 = copy.deepcopy(st)
    res = lr.ppo_update(st, b, hp, 0, 2, 0.2)
    assert torch.equal(res["epoch_start"][0][0], theta_a) and torch.equal(res["epoch_start"][0][1], theta_c)
    for epoch in (0, -1):
        assert lr.ppo_kink_risk(st0, b, hp, res, 0.2, epoch) == 0.0
    b1 = lr.split_net(res["epoch_start"][0][0], D, A)[1]   # agent 0's actor biases of layer 1 (zero-initialised)
    b1[7] = 1e-7
    assert lr.ppo_kink_risk(st0, b, hp, res, 0.2, 0) > 0.0


@pytest.mark.gpu
@pytest.mark.parametrize("sharing,P,n_agents,clip,epochs,lr_", [(False, 64, 2, 0.0, 4, 3e-4), (True, 500, 2, 0.5, 4, 3e-4), ([0, 1, 0], 96, 3, 0.0, 2, 3e-4),
                                                               (False, 128, 2, 0.5, 6, 3e-3)])   # the last: a learning rate that drives ratios out of the clip range
def test_ppo_update_matches_oracle(sharing, P, n_agents, clip, epochs, lr_):
    from codebase_b200.learner import sharing_to_nets
    rng = np.random.default_rng(P + epochs)
    hp = lr.A2CHP(grad_clip=clip, lr=lr_, target_update_interval_or_tau=2)
    m = ac_model(hp, n_agents, D, P, T, sharing=sharing, cls="PPONetwork", num_epochs=epochs)
    nets = sharing_to_nets(sharing, n_agents)
    st = lr.A2CState(m.theta[: m.n_actor].cpu().clone(), m.theta[m.n_actor:].cpu().clone(), m.theta_tgt.cpu().clone(), nets, nets, D, A)
    for u, step in enumerate((0, 3, 4)):
        s = ac_batch(rng, P, n_agents, T, D)
        want = lr.ppo_update(st, ac_oracle_batch(s), hp, step, epochs, 0.2)
        met = m.metrics_dict(m.update_from_store(traj_store(s, m.device), P, step))
        _close([met["loss"], met["actor_loss"], met["value_loss"], met["entropy"]], [want["loss"], want["actor_loss"], want["value_loss"], want["entropy"]], rtol=2e-5, atol=2e-5)
        d = np.abs(m.theta.cpu().numpy() - np.concatenate([st.actor.numpy(), st.critic.numpy()]))
        assert np.quantile(d, 0.999) < 1e-5 * max(1.0, lr_ / 3e-4) and d.max() < 2 * hp.lr * epochs * (u + 1) + 1e-6, (np.quantile(d, 0.999), d.max())
        assert np.quantile(np.abs(m.theta_tgt.cpu().numpy() - st.target.numpy()), 0.999) < 1e-5 * max(1.0, lr_ / 3e-4)
        # keep the two trajectories glued so that later updates compare like for like
        m.theta.copy_(torch.cat([st.actor, st.critic])); m.theta_tgt.copy_(st.target)
        m.adam_m.copy_(torch.cat([st.m["actor"], st.m["critic"]])); m.adam_v.copy_(torch.cat([st.v["actor"], st.v["critic"]]))


@pytest.mark.gpu
@pytest.mark.parametrize("cls", ["A2CNetwork", "PPONetwork"])
def test_standardise_returns_matches_oracle(cls):
    """cfg.standardise_returns=True on the device (marl_a2c_standardise_returns): metrics, running statistics and parameters against the oracle"""
    P, n_agents, epochs = 200, 2, 3
    rng = np.random.default_rng(21)
    hp = lr.A2CHP(target_update_interval_or_tau=2)
    m = ac_model(hp, n_agents, D, P, T, cls=cls, standardise=True, num_epochs=epochs)
    st = lr.A2CState(m.theta[: m.n_actor].cpu().clone(), m.theta[m.n_actor:].cpu().clone(), m.theta_tgt.cpu().clone(), [0, 1], [0, 1], D, A,
                     ret_ms=lr.RunningMeanStdRef((n_agents,)))
    for u, step in enumerate((0, 2, 5)):
        s = ac_batch(rng, P, n_agents, T, D)
        s["rew"] *= 3.0   # returns away from the unit scale the statistics start at
        want = lr.ppo_update(st, ac_oracle_batch(s), hp, step, epochs, 0.2) if cls == "PPONetwork" else lr.a2c_update(st, ac_oracle_batch(s), hp, step)
        met = m.metrics_dict(m.update_from_store(traj_store(s, m.device), P, step))
        _close([met["loss"], met["actor_loss"], met["value_loss"], met["entropy"]], [want["loss"], want["actor_loss"], want["value_loss"], want["entropy"]], rtol=2e-5, atol=2e-5)
        mean, var, count = m.ret_ms()
        _close(mean.numpy(), st.ret_ms.mean.numpy()); _close(var.numpy(), st.ret_ms.var.numpy()); assert abs(count - st.ret_ms.count) < 1e-6
        _, ret, _ = m.scratch(P, T)
        _close(ret.permute(2, 1, 0).cpu().numpy(), want["returns"].numpy(), rtol=2e-5, atol=2e-5)
        d = np.abs(m.theta.cpu().numpy() - np.concatenate([st.actor.numpy(), st.critic.numpy()]))
        assert np.quantile(d, 0.999) < 1e-5, (u, np.quantile(d, 0.999))
        m.theta.copy_(torch.cat([st.actor, st.critic])); m.theta_tgt.copy_(st.target)
        m.adam_m.copy_(torch.cat([st.m["actor"], st.m["critic"]])); m.adam_v.copy_(torch.cat([st.v["actor"], st.v["critic"]]))


@pytest.mark.gpu
@pytest.mark.parametrize("cls,sharing", [("A2CNetwork", False), ("PPONetwork", True)])
def test_centralised_critic_matches_oracle(cls, sharing):
    """MAA2C / MAPPO on the device: the critic passes read the joint observation rows (source mode 2; `values()`: mode 3)"""
    P, n_agents, epochs = 300, 2, 2
    rng = np.random.default_rng(31)
    hp = lr.A2CHP(target_update_interval_or_tau=2)
    m = ac_model(hp, n_agents, D, P, T, sharing=sharing, cls=cls, centralised=True, num_epochs=epochs)
    nets = [0, 0] if sharing else [0, 1]
    assert m.n_critic == len(set(nets)) * lr.net_size(n_agents * D, 1)
    st = lr.A2CState(m.theta[: m.n_actor].cpu().clone(), m.theta[m.n_actor:].cpu().clone(), m.theta_tgt.cpu().clone(), nets, nets, D, A, centralised=True)
    obs = rng.integers(-1, 8, size=(77, n_agents, D)).astype(np.float32)
    joint = torch.tensor(obs.reshape(77, n_agents * D))
    want_v = torch.cat(lr.agents_forward(st.critic, nets, [joint] * n_agents, n_agents * D, 1), -1).numpy()
    _close(m.values(torch.tensor(obs, device="cuda")).cpu().numpy(), want_v)
    for u, step in enumerate((0, 2, 5)):
        s = ac_batch(rng, P, n_agents, T, D)
        want = lr.ppo_update(st, ac_oracle_batch(s), hp, step, epochs, 0.2) if cls == "PPONetwork" else lr.a2c_update(st, ac_oracle_batch(s), hp, step)
        met = m.metrics_dict(m.update_from_store(traj_store(s, m.device), P, step))
        _close([met["loss"], met["actor_loss"], met["value_loss"], met["entropy"]], [want["loss"], want["actor_loss"], want["value_loss"], want["entropy"]], rtol=2e-5, atol=2e-5)
        d = np.abs(m.theta.cpu().numpy() - np.concatenate([st.actor.numpy(), st.critic.numpy()]))
        assert np.quantile(d, 0.999) < 1e-5, (u, np.quantile(d, 0.999))
        m.theta.copy_(torch.cat([st.actor, st.critic])); m.theta_tgt.copy_(st.target)
        m.adam_m.copy_(torch.cat([st.m["actor"], st.m["critic"]])); m.adam_v.copy_(torch.cat([st.v["actor"], st.v["critic"]]))
    sd = m.state_dict()
    assert sd["critic." + ("networks" if sharing else "independent") + ".0.network.0.weight"].shape == (128, n_agents * D)


@pytest.mark.gpu
def test_ippo_driver_runs_and_logs(tmp_path, monkeypatch):
    """ac.train.main with +algorithm=ippo end to end: results.csv has the reference's AC columns"""
    import pandas as pd

    from codebase_b200 import run

    monkeypatch.chdir(tmp_path)
    run.main(["+algorithm=ippo", "env.name=lbforaging:Foraging-8x8-2p-3f-v3", "env.time_limit=25", "env.parallel_envs=256", "seed=1",
              "algorithm.total_steps=40000", "algorithm.eval_interval=10000", f"run_dir={tmp_path}/out"])
    df = pd.read_csv(tmp_path / "out" / "results.csv")
    for col in ("environment_steps", "actor_loss", "entropy", "value_loss", "loss", "mean_episode_returns", "updates"):
        assert col in df.columns, col
    assert len(df) >= 3 and df["environment_steps"].is_monotonic_increasing


@pytest.mark.gpu
@pytest.mark.parametrize("alg", ["maa2c", "mappo"])
def test_centralised_critic_drivers_run_and_log(tmp_path, monkeypatch, alg):
    """+algorithm=maa2c / mappo (critic.centralised: True) end to end on the 2-agent task whose joint observation (30) fits the kernels' 32 input features"""
    import pandas as pd

    from codebase_b200 import run

    monkeypatch.chdir(tmp_path)
    run.main([f"+algorithm={alg}", "env.name=lbforaging:Foraging-8x8-2p-3f-v3", "env.time_limit=25", "env.parallel_envs=256", "seed=2",
              "algorithm.total_steps=30000", "algorithm.eval_interval=10000", f"run_dir={tmp_path}/out"])
    df = pd.read_csv(tmp_path / "out" / "results.csv")
    assert len(df) >= 2 and np.isfinite(df["value_loss"].iloc[-1]) and df["environment_steps"].is_monotonic_increasing

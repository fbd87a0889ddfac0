"""GPU: the fused IA2C learner (marl_a2c_*) against golden vectors produced by the reference's A2CNetwork and against
the CPU oracle on random on-policy batches.  Tolerance 1e-5 (rtol + atol) on float learner tensors."""
import os
import types

import numpy as np
import pytest
import torch

from oracle import learner_ref as lr
from tests.helpers import golden_stride

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
N, D, A, T = 2, 15, 6, 25


def _close(a, b, rtol=1e-5, atol=1e-5):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert np.allclose(a, b, rtol=rtol, atol=atol), float(np.abs(a - b).max())


def _close_scaled(a, b, tol=1e-5):
    """element-wise, relative to the tensor's own scale (Adam's second moment lives at 1e-6 .. 1e-10).  For v = (1 - beta2) g^2 pass tol=2e-5:
    a relative gradient error e shows up as 2e in v, so 2e-5 on v is the 1e-5 bar on g."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    scale = max(float(np.abs(b).max()), 1e-30)
    assert np.abs(a - b).max() <= tol * scale, (float(np.abs(a - b).max()), scale)


def _clipped(grad, max_norm):
    if not max_norm:
        return grad
    norm = float(np.sqrt((grad.astype(np.float64) ** 2).sum()))
    return grad * min(1.0, max_norm / (norm + 1e-6))


def _space(shape=None, n=None):
    return types.SimpleNamespace(shape=shape, n=n)


def _model(sharing, hp, P, n_agents=N):
    from codebase_b200.ac.model import A2CNetwork

    cfg = types.SimpleNamespace(optimizer="Adam", lr=hp.lr, gamma=hp.gamma, grad_clip=hp.grad_clip, n_steps=hp.n_steps, entropy_coef=hp.entropy_coef,
                                value_loss_coef=hp.value_loss_coef, target_update_interval_or_tau=hp.target_update_interval_or_tau, standardise_returns=False)
    net = types.SimpleNamespace(layers=[128, 128], parameter_sharing=sharing, use_rnn=False, use_orthogonal_init=True, centralised=False)
    return A2CNetwork([_space(shape=(D,))] * n_agents, [_space(n=A)] * n_agents, cfg, net, net, "cuda", max_envs=P, max_episode_length=T)


def _to_store(s, device):
    from codebase_b200.lbf import TrajStore

    P, n_agents = s["obs"].shape[0], s["obs"].shape[1]
    ts = TrajStore(P, n_agents, T, D, device)
    for k in ("obs", "act", "rew", "done", "filled"):
        getattr(ts, k).copy_(torch.as_tensor(s[k]))
    return ts


def _oracle_batch(s):
    t = {k: torch.as_tensor(v) for k, v in s.items()}
    P, n_agents = t["obs"].shape[0], t["obs"].shape[1]
    return dict(obss=t["obs"].permute(2, 0, 1, 3).reshape(T + 1, P, n_agents * D).float(), actions=t["act"].permute(2, 0, 1).long(),
                rewards=t["rew"].permute(2, 0, 1).float(), dones=t["done"].permute(1, 0).float(), filled=t["filled"].permute(1, 0).float())


@pytest.mark.parametrize("name", ["ia2c_indep", "ia2c_shared"])
def test_update_matches_reference_golden(name):
    g = np.load(os.path.join(GOLD, f"{name}.npz"))
    hp = lr.A2CHP(lr=float(g["hp"][0]), gamma=float(g["hp"][1]), grad_clip=float(g["hp"][2]), n_steps=int(g["hp"][3]), entropy_coef=float(g["hp"][4]),
                  value_loss_coef=float(g["hp"][5]), target_update_interval_or_tau=float(g["hp"][6]))
    P = g["u0_obs"].shape[0]
    m = _model(bool(int(g["n_nets"]) == 1), hp, P)
    assert m.n_actor == g["actor0"].size and m.n_critic == g["critic0"].size
    m.theta[: m.n_actor].copy_(torch.tensor(g["actor0"])); m.theta[m.n_actor:].copy_(torch.tensor(g["critic0"])); m.theta_tgt.copy_(torch.tensor(g["target0"]))
    for u, step in enumerate(g["steps"]):
        s = {k: g[f"u{u}_{k}"] for k in ("obs", "act", "rew", "done", "filled")}
        met = m.metrics_dict(m.update_from_store(_to_store(s, m.device), P, int(step)))
        _close([met["loss"], met["actor_loss"], met["value_loss"], met["entropy"]], g["metrics"][u])
        if u == 0:
            _, ret, _ = m.scratch(P, T)
            _close(ret.permute(2, 1, 0).cpu().numpy(), g["returns0"])
    S = golden_stride(g)
    am, av = m.adam_m.cpu().numpy(), m.adam_v.cpu().numpy()   # element-wise against the reference optimiser's state
    _close_scaled(am[: m.n_actor][::S], g["actor_adam_m_final"]); _close_scaled(am[m.n_actor:][::S], g["critic_adam_m_final"])
    _close_scaled(av[: m.n_actor][::S], g["actor_adam_v_final"], tol=2e-5); _close_scaled(av[m.n_actor:][::S], g["critic_adam_v_final"], tol=2e-5)
    th, tg = m.theta.cpu().numpy(), m.theta_tgt.cpu().numpy()
    for got, want in ((th[: m.n_actor][::S], g["actor_final"]), (th[m.n_actor:][::S], g["critic_final"]), (tg[::S], g["target_final"])):
        d = np.abs(got - want)
        assert np.quantile(d, 0.999) < 1e-5 and d.max() < 2 * hp.lr * len(g["steps"]) + 1e-6, (np.quantile(d, 0.999), d.max())


@pytest.mark.parametrize("sharing,P,n_agents,clip", [(False, 64, 2, 0.0), (True, 500, 2, 0.5), (False, 1024, 2, 0.0), ([0, 1, 0], 96, 3, 0.0)])
def test_update_matches_oracle_on_random_batches(sharing, P, n_agents, clip):
    from codebase_b200.dqn.model import sharing_to_nets

    rng = np.random.default_rng(P)
    hp = lr.A2CHP(grad_clip=clip)
    m = _model(sharing, hp, P, n_agents)
    nets = sharing_to_nets(sharing, n_agents)
    st = lr.A2CState(m.theta[: m.n_actor].cpu().clone(), m.theta[m.n_actor:].cpu().clone(), m.theta_tgt.cpu().clone(), nets, nets, D, A)
    for u, step in enumerate((0, 3 * P, 200)):
        obs = rng.integers(-1, 8, size=(P, n_agents, T + 1, D)).astype(np.float32)
        act = rng.integers(0, A, size=(P, n_agents, T)).astype(np.int32)
        rew = (rng.random((P, n_agents, T)) < 0.2).astype(np.float32) * rng.random((P, n_agents, T)).astype(np.float32)
        length = rng.integers(1, T + 1, size=P)
        done = np.zeros((P, T + 1), np.uint8); filled = np.zeros((P, T), np.uint8)
        for e in range(P):
            filled[e, : length[e]] = 1
            done[e, length[e]] = 1
        s = dict(obs=obs, act=act, rew=rew, done=done, filled=filled)
        want = lr.a2c_update(st, _oracle_batch(s), hp, step)
        m.update_grads(_to_store(s, m.device), P)
        gr = m.grad.cpu().numpy()
        n = m.n_actor + m.n_critic
        wg = np.concatenate([want["grad"]["actor"].numpy(), want["grad"]["critic"].numpy()])
        scale = max(1.0, float(np.abs(wg).max()))
        _close(gr[:n] / gr[n + 1] / scale, wg / scale)
        _close_scaled(_clipped(gr[:n] / gr[n + 1], clip), np.concatenate([want["grad_clipped"]["actor"].numpy(), want["grad_clipped"]["critic"].numpy()]))
        met = m.metrics_dict(m.update_apply(step))
        _close_scaled(m.adam_m.cpu().numpy(), np.concatenate([st.m["actor"].numpy(), st.m["critic"].numpy()]))
        _close_scaled(m.adam_v.cpu().numpy(), np.concatenate([st.v["actor"].numpy(), st.v["critic"].numpy()]), tol=2e-5)
        _close([met["loss"], met["actor_loss"], met["value_loss"], met["entropy"]], [want["loss"], want["actor_loss"], want["value_loss"], want["entropy"]])
        vt, ret, adv = m.scratch(P, T)
        _close(ret.permute(2, 1, 0).cpu().numpy(), want["returns"].numpy())
        d = np.abs(m.theta.cpu().numpy() - np.concatenate([st.actor.numpy(), st.critic.numpy()]))
        assert np.quantile(d, 0.999) < 1e-5 and d.max() < 2 * hp.lr * (u + 1) + 1e-6
        _close(np.quantile(np.abs(m.theta_tgt.cpu().numpy() - st.target.numpy()), 0.999), 0)
        m.theta.copy_(torch.cat([st.actor, st.critic])); m.theta_tgt.copy_(st.target)
        m.adam_m.copy_(torch.cat([st.m["actor"], st.m["critic"]])); m.adam_v.copy_(torch.cat([st.v["actor"], st.v["critic"]]))


def test_forward_passes_and_reference_style_calls():
    from collections import namedtuple

    rng = np.random.default_rng(1)
    hp = lr.A2CHP()
    P = 300
    m = _model(False, hp, P)
    obs = rng.integers(-1, 8, size=(P, N, D)).astype(np.float32)
    xs = [torch.tensor(obs[:, i]) for i in range(N)]
    _close(m.logits(torch.tensor(obs, device="cuda")).cpu().numpy(), torch.stack(lr.agents_forward(m.theta[: m.n_actor].cpu(), [0, 1], xs, D, A), 1).numpy())
    _close(m.values(torch.tensor(obs, device="cuda")).cpu().numpy(), torch.cat(lr.agents_forward(m.theta[m.n_actor:].cpu(), [0, 1], xs, D, 1), -1).numpy())
    acts, _ = m.act([x.cuda() for x in xs], None)
    assert tuple(acts.shape) == (N, P, 1) and acts.dtype == torch.int64
    # reference-layout Batch through model.update(batch, step)
    Batch = namedtuple("Batch", ["obss", "actions", "rewards", "dones", "filled", "action_masks"])
    st = lr.A2CState(m.theta[: m.n_actor].cpu().clone(), m.theta[m.n_actor:].cpu().clone(), m.theta_tgt.cpu().clone(), [0, 1], [0, 1], D, A)
    Pb = 16
    b = dict(obss=torch.tensor(rng.standard_normal((T + 1, Pb, N * D)), dtype=torch.float32), actions=torch.tensor(rng.integers(0, A, (T, Pb, N))),
             rewards=torch.tensor(rng.random((T, Pb, N)), dtype=torch.float32), dones=torch.tensor(rng.random((T + 1, Pb)) < 0.05, dtype=torch.float32),
             filled=torch.tensor(rng.random((T, Pb)) < 0.9, dtype=torch.float32))
    want = lr.a2c_update(st, b, hp, 7)
    got = m.update(Batch(*[b[k].cuda() for k in ("obss", "actions", "rewards", "dones", "filled")], None), 7)
    _close([got["loss"], got["actor_loss"], got["value_loss"], got["entropy"]], [want["loss"], want["actor_loss"], want["value_loss"], want["entropy"]])
    sd = m.state_dict()
    assert "actor.independent.0.network.0.weight" in sd and sd["critic.independent.1.network.4.weight"].shape == (1, 128) and "target_critic.independent.0.network.2.bias" in sd


def test_ia2c_driver_runs_and_logs(tmp_path, monkeypatch):
    """ac.train.main end to end on a small config: results.csv has the reference's AC columns."""
    import pandas as pd

    from codebase_b200 import run

    monkeypatch.chdir(tmp_path)
    run.main(["+algorithm=ia2c", "env.name=lbforaging:Foraging-8x8-2p-3f-v3", "env.time_limit=25", "env.parallel_envs=256", "seed=1",
              "algorithm.total_steps=40000", "algorithm.eval_interval=10000", f"run_dir={tmp_path}/out"])
    df = pd.read_csv(tmp_path / "out" / "results.csv")
    for col in ("environment_steps", "actor_loss", "entropy", "value_loss", "loss", "mean_episode_returns", "agent0/mean_episode_returns", "mean_episode_length", "updates"):
        assert col in df.columns, col
    assert len(df) >= 3 and df["environment_steps"].is_monotonic_increasing

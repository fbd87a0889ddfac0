"""GPU: observation widths 17..32 (KP = 32 input tiles) -- BASELINE.json configs[3] `Foraging-15x15-4p-5f-v3` has obs = 27,
4 agents.  IDQN / VDN / IA2C updates against the CPU oracle, and the VDN driver end to end on that env."""
import types

import numpy as np
import pytest
import torch

from oracle import learner_ref as lr

from tests.helpers import ac_batch, ac_model, ac_oracle_batch, assert_grad_close, check_margin, redraw_on_near_tie, space, traj_store

pytestmark = pytest.mark.gpu
T, A = 25, 6


def _close(a, b, rtol=1e-5, atol=1e-5):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert np.allclose(a, b, rtol=rtol, atol=atol), float(np.abs(a - b).max())


@pytest.mark.parametrize("mixer,n_agents,D,B", [(0, 4, 27, 96), (1, 4, 27, 300), (0, 2, 17, 64), (0, 3, 32, 40)])
@redraw_on_near_tie
def test_dqn_family_update_wide_obs(mixer, n_agents, D, B):
    from codebase_b200.dqn import model as M

    rng = np.random.default_rng(D * 100 + B)
    hp = lr.DqnHP(mixer=mixer)
    cfg = types.SimpleNamespace(optimizer="Adam", lr=hp.lr, gamma=hp.gamma, grad_clip=hp.grad_clip, double_q=hp.double_q,
                                target_update_interval_or_tau=hp.target_update_interval_or_tau, standardise_returns=False)
    m = (M.VDNetwork if mixer else M.QNetwork)([space(shape=(D,))] * n_agents, [space(n=A)] * n_agents, cfg, [128, 128], False, False, True, "cuda",
                                             max_batch=B, max_episode_length=T)
    st = lr.DqnState(m.theta.cpu().clone(), m.theta_tgt.cpu().clone(), m.agent_net, D, A)
    obs = rng.integers(-1, 15, size=(50, n_agents, D)).astype(np.float32)
    want_q = torch.stack(lr.agents_forward(st.theta, m.agent_net, [torch.tensor(obs[:, i]) for i in range(n_agents)], D, A), 1).numpy()
    _close(m.q_values(torch.tensor(obs, device="cuda")).cpu().numpy(), want_q)
    store = ac_batch(rng, 200, n_agents, T, D, obs_high=15, coop=bool(mixer))
    idx = rng.integers(0, 200, size=B).astype(np.int32)
    batch = lr.batch_from_store(store, idx)
    check_margin(lr, st, batch, hp)   # near-tie in the double-Q argmax: re-drawn by the decorator
    st0 = lr.DqnState(st.theta.clone(), st.theta_tgt.clone(), st.agent_net, st.in_dim, st.out_dim)   # dqn_update steps st in place
    want = lr.dqn_update(st, batch, hp)
    m.update_grads(traj_store(store, m.device), torch.tensor(idx, device="cuda"))
    gr = m.grad.cpu().numpy()
    scale = max(1.0, float(np.abs(want["grad"].numpy()).max()))
    assert_grad_close(lr, st0, batch, hp, gr[: m.n_params] / gr[m.n_params + 1], want["grad"].numpy())   # re-drawn when a ReLU unit on its kink explains the mismatch
    _close(m.update_apply().cpu().numpy()[0], want["loss"])
    d = np.abs(m.theta.cpu().numpy() - st.theta.numpy())
    assert np.quantile(d, 0.999) < 1e-5


def test_a2c_update_wide_obs():
    rng = np.random.default_rng(5)
    n_agents, D, P = 4, 27, 128
    hp = lr.A2CHP()
    m = ac_model(hp, n_agents, D, P, T, sharing=True)
    nets = [0] * n_agents
    st = lr.A2CState(m.theta[: m.n_actor].cpu().clone(), m.theta[m.n_actor:].cpu().clone(), m.theta_tgt.cpu().clone(), nets, nets, D, A)
    s = ac_batch(rng, P, n_agents, T, D, obs_high=15)
    batch = ac_oracle_batch(s)
    want = lr.a2c_update(st, batch, hp, 0)
    met = m.metrics_dict(m.update_from_store(traj_store(s, m.device), P, 0))
    _close([met["loss"], met["actor_loss"], met["value_loss"], met["entropy"]], [want["loss"], want["actor_loss"], want["value_loss"], want["entropy"]])
    d = np.abs(m.theta.cpu().numpy() - np.concatenate([st.actor.numpy(), st.critic.numpy()]))
    assert np.quantile(d, 0.999) < 1e-5


def test_vdn_driver_on_15x15_4p_5f(tmp_path, monkeypatch):
    """BASELINE.json configs[3] shape (smaller env count): VDN + CooperativeReward on Foraging-15x15-4p-5f-v3."""
    import pandas as pd

    from codebase_b200 import run

    monkeypatch.chdir(tmp_path)
    run.main(["+algorithm=vdn", "env.name=lbforaging:Foraging-15x15-4p-5f-v3", "env.time_limit=25", "env.parallel_envs=512", "seed=0",
              "algorithm.total_steps=80000", "algorithm.eval_interval=30000", "algorithm.batch_size=128", "algorithm.buffer_size=4096",
              "algorithm.updates_per_iteration=8", f"run_dir={tmp_path}/out"])
    df = pd.read_csv(tmp_path / "out" / "results.csv")
    assert "agent3/mean_episode_returns" in df.columns and len(df) >= 2 and np.isfinite(df["loss"].iloc[-1])

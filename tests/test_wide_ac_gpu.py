"""GPU: actor-critic inputs of 33..128 features (KP = 64 / 128 input tiles of the FP32 kernels, W1 staged per tile; the GRU kernels' wide
instantiation).  Forward passes, single updates and an unglued MAPPO chain against the oracle, the reference's own numbers
(tests/golden/wide_ac_reference.npz), recurrent parts at those widths, the drivers end to end, and the DQN family's unchanged 32-feature limit."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import learner_ref as lr
from tests import test_ac_chain_gpu as chain
from tests import test_rnn_ac_gpu as rnn
from tests.helpers import STRIDE, ac_model, reference_outputs, traj_store

pytestmark = pytest.mark.gpu


# ---- forward passes ----------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [33, 45, 64, 65, 100, 128])
@pytest.mark.parametrize("E", [37, 20000])
def test_forward_matches_oracle(D, E):
    """logits, values and target values of 2 independent agents at input width D: 37 envs (one ragged tile per CTA) and 20000 (three tiles per
    CTA, the last one ragged: W1 is re-staged for every tile)"""
    torch.manual_seed(D + E)
    m = ac_model(lr.A2CHP(), 2, D, 64, 5)
    m.theta_tgt.copy_(m.theta_tgt + 0.01 * torch.randn_like(m.theta_tgt))
    obs = torch.randint(-1, 9, (E, 2, D)).float()
    xs = [obs[:, i] for i in range(2)]
    for got, flat, out in ((m.logits(obs.cuda()), m.theta[: m.n_actor], 6), (m.values(obs.cuda()), m.theta[m.n_actor:], 1),
                           (m.values(obs.cuda(), target=True), m.theta_tgt, 1)):
        want = torch.stack(lr.agents_forward(flat.cpu(), [0, 1], xs, D, out), 1).reshape(got.shape)
        np.testing.assert_allclose(got.cpu().numpy(), want.numpy(), rtol=1e-5, atol=1e-5 * max(1.0, float(want.abs().max())))
    m.close()


@pytest.mark.parametrize("N,D,sharing", [(4, 27, True), (3, 18, False), (4, 32, [0, 0, 1, 1]), (2, 17, False)])
def test_centralised_values_match_oracle(N, D, sharing):
    """get_value of a centralised critic (joint rows read in place: row-source mode 3) at joint widths 108, 54, 128 and 34"""
    torch.manual_seed(N * D)
    m = ac_model(lr.A2CHP(), N, D, 64, 5, sharing=sharing, centralised=True)
    E = 3001
    obs = torch.randint(-1, 9, (E, N, D)).float()
    joint = obs.reshape(E, N * D)
    for target, flat in ((False, m.theta[m.n_actor:]), (True, m.theta_tgt)):
        want = torch.stack(lr.agents_forward(flat.cpu(), list(m.critic_net), [joint] * N, N * D, 1), 1)[..., 0]
        got = m.values(obs.cuda(), target=target).cpu()
        np.testing.assert_allclose(got.numpy(), want.numpy(), rtol=1e-5, atol=1e-5 * max(1.0, float(want.abs().max())))
    m.close()


# ---- single updates and a chain (the checks of test_ac_chain_gpu.py) ----------------------------------------------------------------------------
Case = chain.Case
ONE = {
    "ia2c3_D45_indep": Case(N=3, D=45, P=256, steps=(0,)),
    "ippo2_D64_shared_clip": Case(ppo=True, N=2, D=64, sharing=True, grad_clip=0.5, steps=(0,), tu=2),
    "maa2c3_D18_joint54": Case(N=3, D=18, centralised=True, P=256, steps=(0,)),
    "mappo4_D27_joint108_shared_standardise": Case(ppo=True, N=4, D=27, sharing=True, centralised=True, standardise=True, steps=(0,), tu=2, epochs=2),
    "maa2c4_D32_joint128_seps": Case(N=4, D=32, sharing=(0, 0, 1, 1), centralised=True, steps=(0,)),
    "mappo2_D17_joint34": Case(ppo=True, N=2, D=17, centralised=True, steps=(0,), tu=2, epochs=2),
}
CHAIN = {
    # six unglued updates, hard target syncs at every even step, running return statistics carried
    "mappo4_D27_joint108_chain": Case(ppo=True, N=4, D=27, centralised=True, standardise=True, steps=(0, 3, 4, 6, 7, 8), tu=2, epochs=2),
}


@pytest.mark.parametrize("case", list(ONE) + list(CHAIN))
def test_update_matches_oracle(case, monkeypatch):
    monkeypatch.setitem(chain.CASES, case, {**ONE, **CHAIN}[case])
    chain.test_chain_matches_oracle(case)


def test_wide_chain_is_deterministic(monkeypatch):
    case = "mappo4_D27_joint108_chain"
    monkeypatch.setitem(chain.CASES, case, CHAIN[case])
    chain.test_chain_is_deterministic(case)


# ---- the reference's own numbers --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key", ["maa2c_shared", "maa2c_indep", "mappo_shared", "mappo_indep", "ia2c_D45"])
def test_fixture_updates_match_reference(key):
    import tests.test_wide_ac as cpu

    g = reference_outputs("wide_ac_reference")
    cls, N, D, _, _, P, steps, clip, sharing, centralised = cpu.REF_CASES[key]
    st, hp = cpu.case_state(key), cpu.case_hp(key)
    m = ac_model(hp, N, D, P, cpu.T, sharing=sharing, cls=cls, centralised=centralised, num_epochs=cpu.EPOCHS)
    m.theta.copy_(torch.cat([st.actor, st.critic])); m.theta_tgt.copy_(st.target)
    for u, (step, s) in enumerate(zip(steps, cpu.case_batches(key))):
        got = m.metrics_dict(m.update_from_store(traj_store(s, m.device), P, step).cpu())
        np.testing.assert_allclose([got[k] for k in cpu.METRICS], g[f"{key}_metrics"][u], rtol=2e-5, atol=2e-5, err_msg=f"update {u}")
    th = m.theta.cpu().numpy()
    for got, name in ((th[: m.n_actor], "actor"), (th[m.n_actor:], "critic"), (m.theta_tgt.cpu().numpy(), "target")):
        d = np.abs(got[::STRIDE] - g[f"{key}_{name}"])
        assert np.quantile(d, 0.999) < 1e-5, (name, float(np.quantile(d, 0.999)))
    m.close()


# ---- recurrent parts at wide inputs ---------------------------------------------------------------------------------------------------------------
RNN_ONE = {
    "maa2c4_D27_rnn_central_critic_joint108": rnn.Case(T=7, N=4, D=27, arnn=False, centralised=True, P=32),
    "ia2c2_D45_rnn_actor": rnn.Case(T=7, N=2, D=45, crnn=False, P=32),
}


@pytest.mark.parametrize("case", list(RNN_ONE))
def test_recurrent_update_matches_oracle(case, monkeypatch):
    monkeypatch.setitem(rnn.ONE, case, RNN_ONE[case])
    rnn.test_single_update_matches_oracle(case)


@pytest.mark.parametrize("sharing,central,N,D,A", [(False, True, 4, 27, 6), (True, False, 2, 45, 6), (False, False, 2, 128, 5)])
def test_recurrent_act_steps_carry_h(sharing, central, N, D, A):
    rnn.test_act_steps_carry_h_like_the_oracle(sharing, central, N, D, A)


# ---- drivers end to end -------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alg,env,extra,N", [
    ("mappo", "Foraging-15x15-4p-5f-v3", [], 4),
    ("maa2c", "Foraging-10x10-3p-3f-v3", ["env.observe_id=True"], 3),
    ("ia2c", "Foraging-20x20-9p-6f-v3", [], 9),
])
def test_driver_runs_at_wide_inputs(alg, env, extra, N, tmp_path, monkeypatch):
    import pandas as pd

    from codebase_b200 import run

    monkeypatch.chdir(tmp_path)
    run.main([f"+algorithm={alg}", f"env.name=lbforaging:{env}", "env.time_limit=25", "env.parallel_envs=256", "seed=0", "algorithm.total_steps=50000",
              "algorithm.eval_interval=10000", f"run_dir={tmp_path}/out", *extra])
    df = pd.read_csv(tmp_path / "out" / "results.csv")
    for k in range(N):
        assert f"agent{k}/mean_episode_returns" in df.columns, df.columns.tolist()
    losses = [c for c in df.columns if "loss" in c]
    assert losses and len(df) >= 2 and all(np.isfinite(df[c].iloc[-1]) for c in losses), df[losses].tail()


# ---- the DQN family keeps its limit -------------------------------------------------------------------------------------------------------------
def test_dqn_create_still_refuses_33():
    from codebase_b200 import _native as nat

    lib = nat.lib()
    cfg = nat.MlpCfg(2, 2, (C.c_int32 * 32)(0, 1), 33, 128, 6)
    hp = nat.DqnHP(3e-4, 0.99, 1.0, 1, 200.0, 0.9, 0.999, 1e-8, 0)
    h = C.c_void_p()
    with pytest.raises(nat.NativeError, match=r"learner kernels: observation width 33 not supported \(1\.\.32\)"):
        nat.check(lib.marl_dqn_create(C.byref(cfg), C.byref(hp), C.c_int32(16), C.c_int32(25), C.c_int32(0), C.byref(h)), "marl_dqn_create")
    with pytest.raises(nat.NativeError, match=r"marl_dqn_create_rnn: obs dim 33 not supported \(1\.\.32\)"):
        nat.check(lib.marl_dqn_create_rnn(C.byref(cfg), C.byref(hp), C.c_int32(16), C.c_int32(25), C.c_int32(0), C.byref(h)), "marl_dqn_create_rnn")
    assert not h.value

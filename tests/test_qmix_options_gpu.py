"""GPU: QMIX with one-layer hypernetworks (`mixing.hypernet_layers=1`) and with `standardise_returns` (csrc/qmix.cuh, csrc/dqn.cu) against the
reference's outputs (tests/golden/qmix_options_reference.npz) and the oracle (tests/qmix_options_ref.py, with oracle/gru_ref.py's recurrent agents): unglued update chains, the
update_n path, recurrent agent networks, the batch-size rule, checkpoints, the training driver and two learners of different shape in one process."""
import copy
import ctypes as C
import dataclasses
import types

import numpy as np
import pytest
import torch

from oracle import gru_ref as gr
from oracle import learner_ref as lr
from oracle import policy_ref
from oracle import qmix_ref as qr
from tests import qmix_options_ref as qo
from tests import test_qmix_options as opts
from tests.helpers import STRIDE, TIE, NearTie, assert_grad_close, random_store, redraw_on_near_tie, reference_outputs, space

pytestmark = pytest.mark.gpu
A = 6
SEED = 0x51A7_0B5E


@dataclasses.dataclass(frozen=True)
class Case:
    hl: int = 1
    N: int = 2
    D: int = 9
    E: int = 64
    T: int = 6
    B: int = 16
    sharing: bool = False
    double_q: bool = True
    tu: float = 2.0
    standardise: bool = False
    rnn: bool = False


def _hp(c):
    return lr.DqnHP(double_q=c.double_q, target_update_interval_or_tau=c.tu)


def _model(c, max_batch=None):
    from codebase_b200.dqn import model as M

    hp = _hp(c)
    cfg = types.SimpleNamespace(optimizer="Adam", lr=hp.lr, gamma=hp.gamma, grad_clip=hp.grad_clip, double_q=c.double_q, target_update_interval_or_tau=c.tu,
                                standardise_returns=c.standardise)
    return M.QMixNetwork([space(shape=(c.D,))] * c.N, [space(n=A)] * c.N, cfg, [128, 128], c.sharing, c.rnn, True,
                         dict(embed_dim=c.E, hypernet_layers=c.hl, hypernet_embed=32), "cuda", max_batch=max_batch or c.B, max_episode_length=c.T)


def _agent_net(c):
    return [0] * c.N if c.sharing else list(range(c.N))


def _oracle(c, m):
    return qo.QmixOptState(m.theta.cpu().clone(), m.theta_tgt.cpu().clone(), m.mix.cpu().clone(), m.mix_tgt.cpu().clone(), _agent_net(c), c.D, A,
                           embed_dim=c.E, hypernet_layers=c.hl, ret_ms=lr.RunningMeanStdRef((1,)) if c.standardise else None)


def _perturb_target(m):
    """a target that differs from the online networks, so that the double-Q pick and the target mixer matter"""
    m.theta_tgt.copy_(m.theta + 0.01 * torch.randn_like(m.theta)); m.mix_tgt.copy_(m.mix + 0.01 * torch.randn_like(m.mix)); m.params_changed()


def _to_store(b, device):
    from codebase_b200.lbf import TrajStore

    n, t1, B, d = b["obss"].shape
    ts = TrajStore(B, n, t1 - 1, d, device)
    ts.obs.copy_(b["obss"].permute(2, 0, 1, 3)); ts.act.copy_(b["actions"].permute(2, 0, 1)); ts.rew.copy_(b["rewards"].permute(2, 0, 1))
    ts.done.copy_(b["dones"].permute(1, 0)); ts.filled.copy_(b["filled"].permute(1, 0))
    return ts


def _close(got, want, tol, what):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    scale = max(1.0, float(np.abs(want).max()))
    err = float(np.abs(got - want).max())
    assert err <= tol * scale, f"{what}: max abs error {err:.3e} > {tol:g} x {scale:.3g}"


def _check_ret_ms(m, st, what):
    mean, var, count = m.ret_ms()
    assert mean.shape == st.ret_ms.mean.shape, (what, mean.shape, st.ret_ms.mean.shape)
    np.testing.assert_allclose(mean.numpy(), st.ret_ms.mean.numpy(), rtol=1e-5, atol=1e-6, err_msg=f"ret_ms mean, {what}")
    np.testing.assert_allclose(var.numpy(), st.ret_ms.var.numpy(), rtol=1e-5, atol=1e-6, err_msg=f"ret_ms var, {what}")
    assert count == pytest.approx(st.ret_ms.count, rel=1e-12), what


def _check_update(c, m, st, st0, b, want, met, hp, what):
    """loss, clip norm, the agents' and the mixer's gradient of one update; then both parameter sets, both targets and the statistics"""
    filled = float(b["filled"].sum())
    assert abs(float(met[0]) - want["loss"]) <= 1e-5 * max(1.0, abs(want["loss"])), f"loss, {what}"
    _close(m.mix_grad[: m.n_mix].cpu().numpy() / filled, want["mix_grad"].numpy(), 2e-5, f"mixer gradient, {what}")
    kink = lambda: qo.qmix_kink_risk(st0, b, hp)
    assert_grad_close(lr, st0, b, hp, m.grad[: m.n_params].cpu().numpy() / filled, want["grad"].numpy(), tol=2e-5, what=f"agents' gradient, {what}", kink_risk=kink)
    assert abs(float(met[1]) - want["grad_norm"]) <= 2e-5 * max(1.0, want["grad_norm"]), f"clip norm, {what}"
    for mine, theirs, name in ((m.theta, st.theta, "theta"), (m.mix, st.mix, "mixer"), (m.theta_tgt, st.theta_tgt, "target"), (m.mix_tgt, st.mix_tgt, "target mixer")):
        assert np.quantile(np.abs(mine.cpu().numpy() - theirs.numpy()), 0.999) < 2e-5, f"{name} after {what}"
    if c.standardise:
        _check_ret_ms(m, st, what)


def _recurrent_kink_risk(st, b, hp):
    with gr.recurrent():
        return qo.qmix_kink_risk(st, b, hp)


def _margin(c, st, b, hp):
    if c.double_q and lr.double_q_margin(lr.DqnState(st.theta, st.theta_tgt, st.agent_net, c.D, A), b, hp) < TIE:
        raise NearTie("double-Q argmax margin")


# ---- 1. the reference's own outputs --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(opts.CASES))
def test_matches_reference_golden(name):
    g, oc = reference_outputs("qmix_options_reference"), opts.CASES[name]
    c = Case(hl=oc.hl, N=oc.N, D=oc.D, B=oc.B, sharing=oc.sharing, tu=oc.tu, standardise=oc.standardise)
    st = opts.seeded_state(oc)
    m = _model(c)
    m.theta.copy_(st.theta); m.theta_tgt.copy_(st.theta_tgt); m.mix.copy_(st.mix); m.mix_tgt.copy_(st.mix_tgt); m.params_changed()
    rng = np.random.default_rng(oc.seed)
    idx = torch.arange(c.B, dtype=torch.int32, device=m.device)
    for u in range(3):
        loss = float(m.update_from_store(_to_store(opts.batch(rng, oc), m.device), idx)[0].item())
        want = float(g[f"{name}_loss"][u])
        assert abs(loss - want) <= 1e-5 * max(1.0, abs(want)), f"loss of update {u}: {loss} vs {want}"
    for mine, key in ((m.theta, "theta"), (m.theta_tgt, "theta_tgt"), (m.mix, "mix"), (m.mix_tgt, "mix_tgt")):
        assert np.quantile(np.abs(mine.cpu().numpy()[::STRIDE] - g[f"{name}_{key}"]), 0.999) < 2e-5, key
    if c.standardise:
        mean, var, count = m.ret_ms()
        np.testing.assert_allclose(mean.numpy(), g[f"{name}_ret_mean"], rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(var.numpy(), g[f"{name}_ret_var"], rtol=1e-5, atol=1e-6)
        assert count == pytest.approx(float(g[f"{name}_ret_count"]), rel=1e-12)
    m.close()


# ---- 2. unglued update chains against the oracle -------------------------------------------------------------------------------------------------
CHAIN = {
    "h1_n2_d9_e64": Case(hl=1, N=2, D=9, E=64, T=6, B=16),
    "h1_n3_d15_e36_shared_polyak": Case(hl=1, N=3, D=15, E=36, T=25, B=33, sharing=True, tu=0.05),
    "h1_n4_d27_e64_single_q": Case(hl=1, N=4, D=27, E=64, T=25, B=21, double_q=False, tu=200.0),
    "h1_n4_d27_e36_hard": Case(hl=1, N=4, D=27, E=36, T=6, B=9, tu=2.0),
    "h1_std_n2_d15_polyak": Case(hl=1, N=2, D=15, E=64, T=25, B=17, standardise=True, tu=0.05),
    "h2_std_n3_d9_shared": Case(hl=2, N=3, D=9, E=64, T=6, B=19, sharing=True, standardise=True),
    "h1_std_n4_d27_single_q": Case(hl=1, N=4, D=27, E=64, T=6, B=11, double_q=False, standardise=True, tu=3.0),
    # above 64 batch entries: ret_moments_cols_kernel takes the moments of the 128 statistics columns, for either mixer
    "h1_std_b128_single_q": Case(hl=1, N=2, D=9, E=64, T=10, B=128, double_q=False, standardise=True, tu=3.0),
    "h2_std_b128_single_q": Case(hl=2, N=2, D=9, E=64, T=10, B=128, double_q=False, standardise=True, tu=3.0),
}


@pytest.mark.parametrize("name", list(CHAIN))
@redraw_on_near_tie
def test_unglued_chain_matches_oracle(name):
    """three updates through marl_dqn_update on ragged episodes; the device state is never re-synchronised with the oracle, which takes the same
    batches in step"""
    c = CHAIN[name]
    hp = _hp(c)
    m = _model(c)
    _perturb_target(m)
    st = _oracle(c, m)
    idx = torch.arange(c.B, dtype=torch.int32, device=m.device)
    for u in range(3):
        b = qr.random_batch(c.N, c.T, c.B, c.D, A, seed=1000 * u + c.B, ragged=True)
        _margin(c, st, b, hp)
        st0 = copy.deepcopy(st)
        want = qo.qmix_update(st, b, hp)
        met = m.update_from_store(_to_store(b, m.device), idx).cpu()
        _check_update(c, m, st, st0, b, want, met, hp, f"update {u}")
    m.close()


# ---- 3. update_n: the loop it replaces, bit for bit, and the oracle ------------------------------------------------------------------------------
UPDATE_N = {
    "h1": Case(hl=1, N=3, D=9, T=10, B=32, tu=3.0),
    "h1_std": Case(hl=1, N=2, D=15, T=10, B=24, standardise=True, tu=0.05),
    "h2_std": Case(hl=2, N=2, D=9, T=10, B=24, standardise=True, tu=3.0),
}


def _state(m):
    out = dict(theta=m.theta, theta_tgt=m.theta_tgt, adam_m=m.adam_m, adam_v=m.adam_v, grad=m.grad, metrics=m._metrics, mix=m.mix, mix_tgt=m.mix_tgt,
               mix_m=m.mix_m, mix_v=m.mix_v, mix_grad=m.mix_grad)
    out = {k: v.detach().cpu().clone() for k, v in out.items()}
    if m.standardise_returns:
        mean, var, count = m.ret_ms()
        out.update(ret_mean=mean, ret_var=var, ret_count=torch.tensor(count, dtype=torch.float64))
    return out


@pytest.mark.parametrize("name", list(UPDATE_N))
@redraw_on_near_tie
def test_update_n_is_the_loop_it_replaces_and_tracks_the_oracle(name):
    from codebase_b200 import _native as nat

    c, K, cap = UPDATE_N[name], 4, 64
    hp = _hp(c)
    a, b = _model(c), _model(c)
    _perturb_target(a)
    for k in ("theta", "theta_tgt", "mix", "mix_tgt"):
        getattr(b, k).copy_(getattr(a, k))
    b.params_changed()
    st = _oracle(c, a)
    store = random_store(np.random.default_rng(c.B), cap, c.N, c.T, c.D, True, A=A)
    from codebase_b200.lbf import TrajStore

    ts = TrajStore(cap, c.N, c.T, c.D, a.device)
    for k in ("obs", "act", "rew", "done", "filled"):
        getattr(ts, k).copy_(torch.as_tensor(store[k]))
    a.update_n(ts, c.B, cap, SEED, 0, K)
    idx = torch.zeros(c.B, dtype=torch.int32, device=b.device)
    for u in range(K):
        nat.check(nat.lib().marl_replay_sample(C.c_uint64(SEED), C.c_uint64(u), C.c_int32(c.B), C.c_int32(cap), nat.ptr(idx), nat.stream_ptr()), "marl_replay_sample")
        ids = policy_ref.replay_sample(SEED, u, c.B, cap)
        assert np.array_equal(idx.cpu().numpy(), ids), f"replay indices of update {u}"
        batch = lr.batch_from_store(store, ids)
        _margin(c, st, batch, hp)
        st0 = copy.deepcopy(st)
        want = qo.qmix_update(st, batch, hp)
        met = b.update_from_store(ts, idx).cpu()
        _check_update(c, b, st, st0, batch, want, met, hp, f"update {u}")
    got, ref = _state(a), _state(b)
    assert got.keys() == ref.keys()
    for k in ref:
        assert torch.equal(got[k], ref[k]), f"{k}: max abs difference {float((got[k].double() - ref[k].double()).abs().max()):.3e}"
    assert a.updates == b.updates == K
    a.close(); b.close()


# ---- 4. recurrent agent networks -----------------------------------------------------------------------------------------------------------------
RNN = {
    "rnn_h1": Case(hl=1, N=2, D=15, T=7, B=13, rnn=True, tu=3.0),
    "rnn_h1_std_shared": Case(hl=1, N=3, D=9, T=7, B=11, rnn=True, sharing=True, standardise=True, tu=0.05),
    "rnn_h2_std": Case(hl=2, N=2, D=15, T=7, B=13, rnn=True, standardise=True, tu=3.0),
}


@pytest.mark.parametrize("name", list(RNN))
@redraw_on_near_tie
def test_recurrent_agents_match_the_oracle(name):
    """use_rnn=True goes through the same mixer branch: loss, gradients and the statistics of every update against oracle/gru_ref.py; the
    parameters at the end, except where Adam's first steps follow the sign of a near-zero gradient (tests/test_rnn_dqn_gpu.py's rule)"""
    from tests.test_rnn_dqn_gpu import _assert_params

    c = RNN[name]
    hp = _hp(c)
    m = _model(c)
    _perturb_target(m)
    st = _oracle(c, m)
    idx = torch.arange(c.B, dtype=torch.int32, device=m.device)
    grads, mgrads = [], []
    for u in range(3):
        b = qr.random_batch(c.N, c.T, c.B, c.D, A, seed=77 * u + c.B, ragged=True)
        if c.double_q:
            with gr.recurrent():
                _margin(c, st, b, hp)
        st0 = copy.deepcopy(st)
        with gr.recurrent():
            want = qo.qmix_update(st, b, hp)
        grads.append(want["grad"]); mgrads.append(want["mix_grad"])
        met = m.update_from_store(_to_store(b, m.device), idx).cpu()
        filled = float(b["filled"].sum())
        assert abs(float(met[0]) - want["loss"]) <= 1e-5 * max(1.0, abs(want["loss"])), f"loss, update {u}"
        _close(m.mix_grad[: m.n_mix].cpu().numpy() / filled, want["mix_grad"].numpy(), 2e-5, f"mixer gradient, update {u}")
        assert_grad_close(lr, st0, b, hp, m.grad[: m.n_params].cpu().numpy() / filled, want["grad"].numpy(), tol=2e-5, what=f"agents' gradient, update {u}",
                          kink_risk=lambda: _recurrent_kink_risk(st0, b, hp))
        if c.standardise:
            _check_ret_ms(m, st, f"update {u}")
    _assert_params(m.theta.cpu().numpy(), st.theta, grads, "theta")
    _assert_params(m.mix.cpu().numpy(), st.mix, mgrads, "mixer")
    m.close()


# ---- 5. the batch-size rule, checkpoints -----------------------------------------------------------------------------------------------------------
def test_standardised_learner_refuses_a_smaller_batch():
    from codebase_b200 import _native as nat

    c = Case(hl=1, B=8, standardise=True)
    m = _model(c)
    ts = _to_store(qr.random_batch(c.N, c.T, 8, c.D, A, seed=4), m.device)
    with pytest.raises(nat.NativeError, match="batch 7 must stay at max_batch 8"):
        m.update_from_store(ts, torch.arange(7, dtype=torch.int32, device=m.device))
    assert np.isfinite(float(m.update_from_store(ts, torch.arange(8, dtype=torch.int32, device=m.device))[0].item()))
    m.close()


def test_one_layer_state_dict_uses_the_reference_keys_and_round_trips():
    c = Case(hl=1, N=2, D=15, T=25, B=32, tu=0.01, standardise=True)
    m = _model(c)
    ts = _to_store(qr.random_batch(c.N, c.T, 64, c.D, A, seed=9), m.device)
    mix0 = m.mix.clone()
    met = m.update_n(ts, 32, 64, 1234, 0, 5).cpu()
    assert m.updates == 5 and np.isfinite(float(met[0])) and float((m.mix - mix0).abs().max()) > 0 and float((m.mix_tgt - mix0).abs().max()) > 0
    sd = m.state_dict()
    mk = sorted(k for k in sd if k.startswith("mixer."))
    assert mk == sorted(f"mixer.{k}.{p}" for k in ("hyper_w_1", "hyper_w_final", "hyper_b_1", "V.0", "V.2") for p in ("weight", "bias"))
    assert sd["mixer.hyper_w_1.weight"].shape == (2 * 64, 30) and sd["target_mixer.hyper_w_final.weight"].shape == (64, 30) and sd["mixer.V.2.bias"].shape == (1,)
    m2 = _model(c)
    m2.load_state_dict(sd)
    assert torch.equal(m2.mix, m.mix) and torch.equal(m2.mix_tgt, m.mix_tgt) and torch.equal(m2.theta, m.theta) and torch.equal(m2.theta_tgt, m.theta_tgt)
    m.close(); m2.close()


# ---- 6. the training driver, checkpoint -> eval ------------------------------------------------------------------------------------------------------
def _driver(tmp_path, monkeypatch, env, extra, updates_per_iteration=16, finite_loss=True):
    import pandas as pd

    from codebase_b200 import run

    monkeypatch.chdir(tmp_path)
    out = f"{tmp_path}/out"
    run.main(["+algorithm=qmix", f"env.name={env}", "env.time_limit=25", "env.parallel_envs=256", "seed=0", "algorithm.total_steps=60000",
              "algorithm.eval_interval=20000", "algorithm.save_interval=15000", "algorithm.batch_size=128", "algorithm.buffer_size=4096",
              f"algorithm.updates_per_iteration={updates_per_iteration}", f"run_dir={out}"] + extra)
    df = pd.read_csv(f"{out}/results.csv")
    assert list(df.columns)[0] == "environment_steps" and "loss" in df.columns
    assert len(df) >= 2 and df["updates"].iloc[-1] > 0 and (np.isfinite(df["loss"].iloc[-1]) or not finite_loss)
    return out


def test_driver_one_layer_standardised_and_eval(tmp_path, monkeypatch):
    """The driver trains with both options and its checkpoint plays in codebase_b200.eval.  The loss value is not asserted: the reference's
    de-standardised target (Q' sqrt(var) + mean) feeds the running variance back into the next returns, and on untrained networks that loop grows
    the statistics geometrically (tests/qmix_options_ref.py reaches an infinite variance after ~20 updates of random episodes; this run's loss was NaN
    after 8 updates).  The arithmetic of each update is pinned against the oracle and the reference above.  This run's batch of 128 takes
    ret_moments_cols_kernel for the statistics' moments; that kernel is not the cause: tests/test_td_target_edges_gpu.py holds its running
    statistics and standardised returns to float64 at 65 and 128 batch entries, and the B = 128 cases of CHAIN hold whole standardised updates to
    the oracle."""
    import os

    from codebase_b200 import eval as ev

    out = _driver(tmp_path, monkeypatch, "lbforaging:Foraging-8x8-2p-3f-v3", ["algorithm.model.mixing.hypernet_layers=1", "algorithm.standardise_returns=True"],
                  finite_loss=False)
    steps = sorted(int(f[7:-3]) for f in os.listdir(f"{out}/checkpoints"))
    sd = torch.load(f"{out}/checkpoints/model_s{steps[-1]}.pt", weights_only=True)
    assert "target_mixer.hyper_w_1.weight" in sd and "mixer.hyper_w_1.0.weight" not in sd
    monkeypatch.chdir(tmp_path)
    res = ev.main([f"path={out}", "episodes=64", "seed=3"])
    assert res["load_step"] == steps[-1] and res["episodes"] == 64 and np.isfinite(res["mean_episode_returns"])


def test_driver_one_layer_on_15x15_4p_5f(tmp_path, monkeypatch):
    _driver(tmp_path, monkeypatch, "lbforaging:Foraging-15x15-4p-5f-v3", ["algorithm.model.mixing.hypernet_layers=1"])


# ---- 7. two learners of different shape in one process -------------------------------------------------------------------------------------------
def test_one_layer_four_agent_and_two_layer_two_agent_learners_coexist():
    """qmix_mix_kernel's shared-memory opt-in is per function instantiation and process-wide: the 4-agent one-layer learner (164 KB) and the 2-agent
    two-layer learner alternate updates, each against its own oracle"""
    big_c, small_c = Case(hl=1, N=4, D=27, B=8), Case(hl=2, N=2, D=9, B=8)
    big, small = _model(big_c), _model(small_c)
    states = {id(big): _oracle(big_c, big), id(small): _oracle(small_c, small)}
    idx = torch.arange(8, dtype=torch.int32, device=big.device)
    for u, (m, c) in enumerate(((small, small_c), (big, big_c), (small, small_c), (big, big_c))):
        b = qr.random_batch(c.N, c.T, 8, c.D, A, seed=50 + u)
        st = states[id(m)]
        st0 = copy.deepcopy(st)
        want = qo.qmix_update(st, b, _hp(c))
        met = m.update_from_store(_to_store(b, m.device), idx).cpu()
        assert np.isfinite(float(met[0])) and float(met[4]) > 0
        if lr.double_q_margin(lr.DqnState(st0.theta, st0.theta_tgt, st0.agent_net, c.D, A), b, _hp(c)) >= TIE:
            assert abs(float(met[0]) - want["loss"]) <= 1e-5 * max(1.0, abs(want["loss"])), f"loss of update {u}"
    big.close(); small.close()

"""GPU: recurrent (GRU) agent networks of IDQN / VDN / QMIX (csrc/gru_kernels.cu behind marl_dqn_create_rnn) against the oracle restatement
(oracle/gru_ref.py, itself pinned to the reference's outputs by test_rnn_dqn.py): the act step carrying h, single updates on ragged stores,
the goldens, unglued update_n chains, bit-for-bit determinism of the three update forms, and the training driver end to end."""
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
from tests.helpers import NearTie, TIE, assert_grad_close, close_scaled, random_store, redraw_on_near_tie, space, traj_store

pytestmark = pytest.mark.gpu
MIXING = dict(embed_dim=64, hypernet_layers=2, hypernet_embed=32)
SEED = 0x0DD5_EED5


@dataclasses.dataclass(frozen=True)
class Case:
    mixer: int = 0
    N: int = 2
    D: int = 15
    A: int = 6
    sharing: object = False
    B: int = 37
    T: int = 7
    tu: float = 3.0
    grad_clip: float = 1.0
    double_q: bool = True
    standardise: bool = False
    cap: int = 64


def _hp(c):
    return lr.DqnHP(grad_clip=c.grad_clip or 0.0, double_q=c.double_q, target_update_interval_or_tau=c.tu, mixer=min(c.mixer, 1))


def _agent_net(c):
    from codebase_b200.learner import sharing_to_nets

    return sharing_to_nets(c.sharing, c.N)


def _learner(c):
    from codebase_b200.dqn import model as M

    hp = _hp(c)
    cfg = types.SimpleNamespace(optimizer="Adam", lr=hp.lr, gamma=hp.gamma, grad_clip=c.grad_clip, double_q=c.double_q, target_update_interval_or_tau=c.tu,
                                standardise_returns=c.standardise)
    args = ([space(shape=(c.D,))] * c.N, [space(n=c.A)] * c.N, cfg, [128, 128], c.sharing, True, True)
    if c.mixer == 2:
        return M.QMixNetwork(*args, MIXING, "cuda", max_batch=c.B, max_episode_length=c.T)
    return (M.VDNetwork if c.mixer else M.QNetwork)(*args, "cuda", max_batch=c.B, max_episode_length=c.T)


def _oracle(c, m):
    th = m.theta.detach().cpu().clone()
    if c.mixer == 2:
        mx = m.mix.detach().cpu().clone()
        return qr.QmixState(th, m.theta_tgt.detach().cpu().clone(), mx, m.mix_tgt.detach().cpu().clone(), _agent_net(c), c.D, c.A)
    st = lr.DqnState(th, m.theta_tgt.detach().cpu().clone(), _agent_net(c), c.D, c.A)
    if c.standardise:
        st.ret_ms = lr.RunningMeanStdRef((1,) if c.mixer == 1 else (c.N,))
    return st


def _store(c, seed):
    s = random_store(np.random.default_rng(seed), c.cap, c.N, c.T, c.D, c.mixer != 0, A=c.A)
    s["obs"] = (s["obs"] / 6.0).astype(np.float32)
    return s


def _check_tie(c, st, batch, hp):
    if c.double_q and c.mixer != 2 and gr.double_q_margin(st, batch, hp) < TIE:
        raise NearTie("double-Q argmax margin")


def _kink(c, st, batch, hp):
    return (lambda: gr.qmix_kink_risk(st, batch, hp)) if c.mixer == 2 else (lambda: gr.dqn_kink_risk(st, batch, hp))


def _oracle_update(c, st, batch, hp):
    return gr.qmix_update(st, batch, hp) if c.mixer == 2 else gr.dqn_update(st, batch, hp)


def _assert_params(got, st_theta, grads, what, tol=1e-5):
    """parameters to tol, except elements whose oracle gradient stayed below 1e-4 of the largest on some step (Adam's first steps move them by
    ~lr x sign(g): the sign of a near-zero gradient is not determined by either implementation).  At T = 1 that is all of W_hh: the
    zero initial state gives it no gradient."""
    got, want = np.asarray(got, np.float64), st_theta.numpy().astype(np.float64)
    ok = np.ones_like(want, bool)
    for g in grads:
        g = np.abs(g.numpy())
        ok &= g >= 1e-4 * g.max()
    err = np.abs(got - want)[ok]
    assert ok.any() and float(err.max()) <= tol, (what, float(err.max()), float(ok.mean()))


# ---- 1. the act step ----------------------------------------------------------------------------------------------------------------------------
ACT = [(False, 15, 6), (True, 17, 3), ([0, 0, 1], 27, 8), (False, 32, 8), (True, 15, 6), ([0, 0, 1], 32, 3)]


@pytest.mark.parametrize("sharing,D,A", ACT)
def test_act_step_carries_h_like_the_oracle(sharing, D, A):
    """S steps of marl_dqn_forward_rnn, each fed the previous h_out, equal the oracle's recurrence at every step (Q and h); h_in = NULL and
    explicit zeros give bit-equal results; the target network is used when asked"""
    N = 3 if isinstance(sharing, list) else 2
    c = Case(N=N, D=D, A=A, sharing=sharing, B=8, T=4)
    torch.manual_seed(D * 10 + A)
    m = _learner(c)
    m.theta_tgt.copy_(m.theta + 0.05 * torch.randn_like(m.theta)); m.params_changed()
    E, S = 37, 12
    obs = (torch.randint(-1, 12, (S, E, N, D)) / 6.0).float()
    want_q, want_h = gr.act_steps(m.theta.cpu(), _agent_net(c), obs, D, A)
    h = None
    for s in range(S):
        q, h_new = m.q_values(obs[s].cuda().contiguous(), h=h)
        np.testing.assert_allclose(q.cpu().numpy(), want_q[s].numpy(), rtol=0, atol=1e-5 * max(1.0, float(want_q[s].abs().max())), err_msg=f"q step {s}")
        np.testing.assert_allclose(h_new.cpu().numpy(), want_h[s].numpy(), rtol=0, atol=1e-5, err_msg=f"h step {s}")
        h = h_new.clone()
    q0, h0 = m.q_values(obs[0].cuda().contiguous(), h=None)
    q1, h1 = m.q_values(obs[0].cuda().contiguous(), h=torch.zeros(E, N, 128, device="cuda"))
    assert torch.equal(q0, q1) and torch.equal(h0, h1)
    qt, _ = m.q_values(obs[0].cuda().contiguous(), target=True)
    want_t, _ = gr.act_steps(m.theta_tgt.cpu(), _agent_net(c), obs[:1], D, A)
    np.testing.assert_allclose(qt.cpu().numpy(), want_t[0].numpy(), rtol=0, atol=1e-5 * max(1.0, float(want_t.abs().max())))
    from codebase_b200 import _native as nat
    with pytest.raises(nat.NativeError, match="marl_dqn_forward_rnn"):
        nat.check(m._lib.marl_dqn_forward(m._h, nat.ptr(obs[0].cuda().contiguous()), C.c_int32(E), C.c_int32(0), nat.ptr(q0), nat.stream_ptr()), "marl_dqn_forward")
    with pytest.raises(nat.NativeError, match="alias"):
        m.q_values(obs[0].cuda().contiguous(), h=h0, h_out=h0)
    m.close()


# ---- 2. single updates against the oracle ------------------------------------------------------------------------------------------------------
ONE = {
    "idqn_T1": Case(T=1, B=37),
    "idqn_T7_shared_polyak_noclip": Case(T=7, B=37, sharing=True, tu=0.05, grad_clip=None, double_q=False),
    "idqn_T25_N4_seps": Case(T=25, B=21, N=4, sharing=[0, 1, 1, 0], D=17, A=8),
    "idqn_T50_N1": Case(T=50, B=19, N=1, A=3),
    "idqn_standardise": Case(T=7, B=37, standardise=True),
    "vdn_T25": Case(mixer=1, T=25, B=37),
    "vdn_standardise_T7": Case(mixer=1, T=7, B=37, standardise=True, grad_clip=None),
    "qmix_T7_shared": Case(mixer=2, T=7, B=37, sharing=True),
    "qmix_T25_N4": Case(mixer=2, T=25, B=21, N=4),
}


@pytest.mark.parametrize("case", list(ONE))
@redraw_on_near_tie
def test_single_update_matches_oracle(case):
    """update_grads: loss and gradient (BPTT) against the oracle; update_apply: Adam m / v and the parameters"""
    c = ONE[case]
    m = _learner(c)
    m.theta_tgt.copy_(m.theta + 0.02 * torch.randn_like(m.theta)); m.params_changed()
    st, hp = _oracle(c, m), _hp(c)
    s = _store(c, int(torch.randint(0, 1 << 30, (1,))))
    ts = traj_store(s, m.device)
    idx = torch.randint(0, c.cap, (c.B,), dtype=torch.int32)
    batch = lr.batch_from_store(s, idx.numpy())
    _check_tie(c, st, batch, hp)
    st0 = copy.deepcopy(st)
    res = _oracle_update(c, st, batch, hp)
    m.update_grads(ts, idx.cuda())
    g = m.grad.cpu().double()
    n = m.n_params
    filled = float(g[n + 1])
    assert filled == float(batch["filled"].sum())
    assert abs(float(g[n]) / filled - res["loss"]) <= 1e-5 * max(1.0, abs(res["loss"]))
    assert_grad_close(lr, st0, batch, hp, (g[:n] / filled).numpy(), res["grad"].numpy(), what=case, kink_risk=_kink(c, st0, batch, hp))
    met = m.update_apply().cpu()
    assert abs(float(met[0]) - res["loss"]) <= 1e-5 * max(1.0, abs(res["loss"]))
    gc = res.get("grad_clipped", res["grad"] * (lr.clip_coef(res["grad"], hp.grad_clip)[0] if hp.grad_clip else 1.0))
    # relative to each tensor's largest element: the gradient sums over up to 26 steps x B sequences in another order than the oracle's autograd
    # (~3e-5 of the largest |g| seen on T = 25; the gradient itself meets the 1e-5 bar above), and v = (1 - beta2) g^2 doubles that
    close_scaled(m.adam_m.cpu().numpy(), st.m.numpy(), 5e-5)
    close_scaled(m.adam_v.cpu().numpy(), st.v.numpy(), 1e-4)
    _assert_params(m.theta.cpu().numpy(), st.theta, [gc], case)
    if c.standardise:
        mean, var, count = m.ret_ms()   # one column per agent (VDN: per batch entry)
        np.testing.assert_allclose(mean.numpy(), st.ret_ms.mean.numpy().reshape(-1), rtol=1e-4, atol=1e-6)
        np.testing.assert_allclose(var.numpy(), st.ret_ms.var.numpy().reshape(-1), rtol=1e-4, atol=1e-6)
        assert abs(count - st.ret_ms.count) < 1e-6 * count
    m.close()


# ---- 3. the goldens (the reference's own numbers) ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["idqn_indep", "idqn_shared", "vdn_indep", "qmix_shared", "idqn_standardise"])
def test_three_updates_match_reference_golden(name):
    import tests.test_rnn_dqn as cpu

    g = np.load(cpu.golden_path(name))
    mixer, sharing, kw, standardise, _ = cpu.CASES[name]
    hp, agent_net, n_nets, theta0, mix0, _, _, _ = cpu.case_setup(name)
    c = Case(mixer=mixer, N=cpu.N, D=cpu.D, A=cpu.A, sharing=sharing, B=cpu.B, T=cpu.T, tu=kw["target_update_interval_or_tau"],
             grad_clip=kw["grad_clip"] or None, double_q=kw["double_q"], standardise=standardise, cap=cpu.CAP)
    m = _learner(c)
    m.theta.copy_(theta0); m.theta_tgt.copy_(theta0)
    if mixer == 2:
        m.mix.copy_(mix0); m.mix_tgt.copy_(mix0)
    m.params_changed()
    ts = traj_store({k: g[f"store_{k}"] for k in ("obs", "act", "rew", "done", "filled")}, m.device)
    for u in range(3):
        met = m.update_from_store(ts, torch.tensor(g["idx"][u]).cuda()).cpu()
        want = float(g["loss"][u])
        assert abs(float(met[0]) - want) <= 1e-5 * max(1.0, abs(want)), (u, float(met[0]), want)
    for got, key in ((m.theta, "theta3"), (m.theta_tgt, "theta_tgt3")):
        assert np.quantile(np.abs(got.cpu().numpy()[::cpu.STRIDE] - g[key]), 0.999) < 1e-5, key
    close_scaled(m.adam_m.cpu().numpy()[::cpu.STRIDE], g["m3"], 3e-5)
    close_scaled(m.adam_v.cpu().numpy()[::cpu.STRIDE], g["v3"], 8e-5)
    m.close()
    m = _learner(c)   # the act steps were recorded at the initial parameters
    m.theta.copy_(theta0); m.params_changed()
    h = None
    for s in range(10):
        q, h_new = m.q_values(torch.tensor(g["act_obs"][s]).view(1, cpu.N, cpu.D).cuda(), h=h)
        np.testing.assert_allclose(q[0].cpu().numpy(), g["act_q"][s], rtol=0, atol=1e-5)
        np.testing.assert_allclose(h_new[0].cpu().numpy(), g["act_h"][s], rtol=0, atol=1e-5)
        h = h_new.clone()
    m.close()


# ---- 4. unglued update_n chains ------------------------------------------------------------------------------------------------------------------
CHAIN = {
    "idqn_hard": Case(B=48, T=25, tu=2.0),
    "vdn_standardise_polyak": Case(mixer=1, B=48, T=25, tu=0.05, standardise=True),
    "qmix_hard": Case(mixer=2, B=48, T=25, tu=3.0),
}


@pytest.mark.parametrize("case", list(CHAIN))
@redraw_on_near_tie
def test_update_n_chain_matches_oracle(case):
    """six updates, one update_n call each (the device draws its own indices and carries Adam, targets, counters and return statistics); the oracle
    takes the same batches in step and is never copied back"""
    from codebase_b200 import _native as nat

    c, K = CHAIN[case], 6
    m = _learner(c)
    st, hp = _oracle(c, m), _hp(c)
    s = _store(c, int(torch.randint(0, 1 << 30, (1,))))
    ts = traj_store(s, m.device)
    idx = torch.zeros(c.B, dtype=torch.int32, device=m.device)
    grads = []
    for u in range(K):
        nat.check(nat.lib().marl_replay_sample(C.c_uint64(SEED), C.c_uint64(u), C.c_int32(c.B), C.c_int32(c.cap), nat.ptr(idx), nat.stream_ptr()), "sample")
        want_idx = policy_ref.replay_sample(SEED, u, c.B, c.cap)
        assert np.array_equal(idx.cpu().numpy(), want_idx), f"replay indices of update {u}"
        batch = lr.batch_from_store(s, want_idx)
        _check_tie(c, st, batch, hp)
        res = _oracle_update(c, st, batch, hp)
        grads.append(res.get("grad_clipped", res["grad"]))
        met = m.update_n(ts, c.B, c.cap, SEED, u, 1).cpu()
        assert abs(float(met[0]) - res["loss"]) <= 2e-5 * max(1.0, abs(res["loss"])), (u, float(met[0]), res["loss"])
        assert m.updates == st.updates == u + 1
        _assert_params(m.theta.cpu().numpy(), st.theta, grads, f"{case} theta after update {u}", tol=2e-5)
        _assert_params(m.theta_tgt.cpu().numpy(), st.theta_tgt, grads, f"{case} target after update {u}", tol=2e-5)
        if c.mixer == 2:
            assert np.quantile(np.abs(m.mix.cpu().numpy() - st.mix.numpy()), 0.999) < 2e-5
        if c.standardise:
            mean, var, count = m.ret_ms()
            assert abs(count - st.ret_ms.count) < 1e-6 * count
            np.testing.assert_allclose(mean.numpy(), st.ret_ms.mean.numpy().reshape(-1), rtol=1e-4, atol=1e-5)
    u_, last = C.c_int64(), C.c_int64()
    nat.check(m._lib.marl_dqn_counters(m._h, C.byref(u_), C.byref(last)), "counters")
    assert (int(u_.value), int(last.value)) == (st.updates, st.last_target_update)
    m.close()


# ---- 5. determinism -----------------------------------------------------------------------------------------------------------------------------
def _state(m):
    out = dict(theta=m.theta, theta_tgt=m.theta_tgt, adam_m=m.adam_m, adam_v=m.adam_v, metrics=m._metrics)
    if m.mixer == 2:
        out.update(mix=m.mix, mix_tgt=m.mix_tgt, mix_m=m.mix_m, mix_v=m.mix_v)
    return {k: v.detach().cpu().clone() for k, v in out.items()}


@pytest.mark.parametrize("mixer", [0, 1, 2])
def test_update_forms_are_bit_identical(mixer):
    """two handles through the same update_n chain and update_n against K x (replay_sample + update): bit for bit.  update_grads + update_apply
    against update: the two-call form reduces the clip norm over the whole gradient (an all-reduce may sit between the calls) instead of the
    fused tail's per-block sums, so the clip coefficient may differ in the last bit: equal to 1e-7."""
    from codebase_b200 import _native as nat

    c, K = Case(mixer=mixer, B=40, T=25, tu=2.0), 5
    torch.manual_seed(5)
    ms = [_learner(c) for _ in range(4)]
    for m in ms[1:]:
        m.theta.copy_(ms[0].theta); m.theta_tgt.copy_(ms[0].theta_tgt)
        if mixer == 2:
            m.mix.copy_(ms[0].mix); m.mix_tgt.copy_(ms[0].mix_tgt)
        m.params_changed()
    ts = traj_store(_store(c, 11), ms[0].device)
    ms[0].update_n(ts, c.B, c.cap, SEED, 0, K)
    ms[1].update_n(ts, c.B, c.cap, SEED, 0, K)
    idx = torch.zeros(c.B, dtype=torch.int32, device=ms[0].device)
    for u in range(K):
        nat.check(nat.lib().marl_replay_sample(C.c_uint64(SEED), C.c_uint64(u), C.c_int32(c.B), C.c_int32(c.cap), nat.ptr(idx), nat.stream_ptr()), "sample")
        ms[2].update_from_store(ts, idx)
        ms[3].update_grads(ts, idx); ms[3].update_apply()
    ref = _state(ms[0])
    for i, m in enumerate(ms[1:], 1):
        got = _state(m)
        for k in ref:
            if i < 3:
                assert torch.equal(got[k], ref[k]), (i, k)
            else:
                assert torch.allclose(got[k], ref[k], rtol=1e-6, atol=1e-7), (k, float((got[k] - ref[k]).abs().max()))
    for m in ms:
        m.close()


# ---- 6. the training driver ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("env", ["Foraging-8x8-2p-3f-v3", "Foraging-2s-8x8-2p-2f-coop-v3"])
@pytest.mark.parametrize("alg", ["idqn", "vdn", "qmix"])
def test_driver_trains_recurrent_agents(tmp_path, monkeypatch, alg, env):
    import pandas as pd

    from codebase_b200 import run
    from tests.test_dqn_driver_gpu import IDQN_COLS

    monkeypatch.chdir(tmp_path)
    run.main([f"+algorithm={alg}", f"env.name=lbforaging:{env}", "env.time_limit=25", "env.parallel_envs=128", "seed=0", "algorithm.model.use_rnn=True",
              "algorithm.total_steps=20000", "algorithm.eval_interval=6000", "algorithm.batch_size=64", "algorithm.buffer_size=1024",
              "algorithm.updates_per_iteration=4", f"run_dir={tmp_path}/out"])
    df = pd.read_csv(tmp_path / "out" / "results.csv")
    assert list(df.columns) == IDQN_COLS and len(df) >= 2 and df["updates"].iloc[-1] > 0 and np.isfinite(df["loss"].iloc[-1])
    assert df["mean_episode_length"].between(1, 25).all()


def test_checkpoint_eval_round_trip(tmp_path, monkeypatch):
    import os

    from codebase_b200 import eval as ev
    from codebase_b200 import run

    monkeypatch.chdir(tmp_path)
    out = f"{tmp_path}/out"
    run.main(["+algorithm=idqn", "env.name=lbforaging:Foraging-8x8-2p-3f-v3", "env.time_limit=25", "env.parallel_envs=128", "seed=0",
              "algorithm.model.use_rnn=True", "algorithm.total_steps=12000", "algorithm.eval_interval=6000", "algorithm.save_interval=5000",
              "algorithm.batch_size=64", "algorithm.buffer_size=1024", "algorithm.updates_per_iteration=4", f"run_dir={out}"])
    monkeypatch.chdir(tmp_path)
    steps = sorted(int(f[7:-3]) for f in os.listdir(f"{out}/checkpoints"))
    sd = torch.load(f"{out}/checkpoints/model_s{steps[-1]}.pt", weights_only=True)
    assert "critic.independent.0.rnn.weight_hh_l0" in sd and tuple(sd["critic.independent.0.rnn.weight_hh_l0"].shape) == (384, 128)
    res = ev.main([f"path={out}", "episodes=32", "seed=3"])
    assert res["load_step"] == steps[-1] and res["episodes"] == 32 and np.isfinite(res["mean_episode_returns"])

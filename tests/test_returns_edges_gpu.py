"""GPU: the actor-critic return pass (`a2c_prepare`, csrc/a2c.cu and csrc/retms.cuh) at the boundaries of its splits, against float64.

a. lambda_returns_kernel at every window and lane boundary (tests/returns_ref.py: windows of 256 steps, lanes of 8; one-step and full windows,
   up to five windows, dones and reward spikes on the edges, both block classes of N·P, N = 32), γ in {0.99, 0.999}, λ in {0, 0.5, 0.95, 1}, raw
   and standardised, against the streamed mixture of tests/gae_ref.py, every row held to |got - want| <= τ S_t; each case twice, bit for bit.
b. nstep_returns_kernel at n_steps in {1, 5, 63, 64} where t + n meets T, against oracle.learner_ref.nstep_returns, with the same per-row bar.
c. Return standardisation (ret_moments_kernel, N <= 32) at P·T on both sides of its grid stride, over three updates, and at returns of mean 50
   and spread 0.01, where FP32 moments would lose the variance.
d. Whole updates at long T against the oracle at the tolerances of tests/test_rnn_ac_gpu.py.
Run with -s to see each sweep's worst err / (τ S_t)."""
import copy

import numpy as np
import pytest
import torch

from oracle import learner_ref as lr
from tests import gae_ref as gr
from tests import gru_ac_ref as gar
from tests import returns_ref as rr
from tests.helpers import TIE, NearTie, ac_model, ac_oracle_batch, redraw_on_near_tie, traj_store
from tests.test_rnn_ac_gpu import Case, Tracker, _batch, _check_update, _hp, _model, _oracle, _perturb_target

pytestmark = pytest.mark.gpu


def _pair(hp, N, P, T, standardise, seed):
    """two handles with the same parameters (the second replays every update: the bits must agree), the target critic moved off the critic"""
    torch.manual_seed(seed)
    a, b = (ac_model(hp, N, rr.D, P, T, A=3, standardise=standardise) for _ in range(2))
    a.theta_tgt.copy_(a.theta_tgt + 0.05 * torch.randn_like(a.theta_tgt))
    b.theta.copy_(a.theta); b.theta_tgt.copy_(a.theta_tgt)
    return a, b


def _target_values(vt, ms):
    """the device's target values [N][P][T+1] as (T+1, P, N) float64, de-standardised with the statistics ms = (mean, var) the update read"""
    v = vt.double().permute(2, 1, 0).numpy()
    if ms is not None:
        v = v * np.sqrt(ms[1].double().numpy()) + ms[0].double().numpy()
    return v


def _check_stats(m, stats, what):
    mean, var, count = m.ret_ms()
    assert count == stats.count, (what, count, stats.count)
    em = np.abs(mean.double().numpy() - stats.mean) / stats.mean_bar
    ev = np.abs(var.double().numpy() - stats.var) / stats.var_bar
    assert em.max() <= 1.0 and ev.max() <= 1.0, f"{what}: running mean at {em.max():.2f}, var at {ev.max():.2f} of their bars"
    return max(float(em.max()), float(ev.max()))


def _standardised_ratio(got, want, S, bar, stats):
    """the standardised returns against (want - mean) / sqrt(var) of the float64 statistics: the returns' bar divided by the spread, plus the
    statistics' own bars carried through the standardisation, plus its float32 roundings"""
    sd = np.sqrt(stats.var)
    z = (want - stats.mean) / sd
    zbar = (bar * S + stats.mean_bar) / sd + (0.5 * stats.var_bar / stats.var + 4 * rr.U32) * np.abs(z)
    return float((np.abs(got - z) / zbar).max())


WORST = {}


def _record(sweep, ratio):
    WORST[sweep] = max(WORST.get(sweep, 0.0), ratio)
    return ratio


# ---- a. λ-returns ----------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("standardise", [False, True], ids=["raw", "standardise"])
@pytest.mark.parametrize("T,N,block", rr.LAMBDA_CASES)
def test_lambda_returns_at_the_split_boundaries(T, N, block, standardise):
    P = rr.case_P(T, N, block)
    s = rr.lambda_batch(np.random.default_rng(T * 7 + N), T, N, P)
    rew, done, _ = rr.sequences(s)
    worst = 0.0
    for gamma in rr.GAMMAS:
        a, b = _pair(lr.A2CHP(gamma=gamma), N, P, T, standardise, T * 31 + N)
        ts = traj_store(s, a.device)
        stats = rr.StatsRef(N) if standardise else None
        for lam in rr.LAMBDAS:
            ms = a.ret_ms()[:2] if standardise else None
            outs = []
            for m in (a, b):
                m.set_gae_lambda(lam)
                m.update_grads(ts, P)
                vt, ret, _ = m.scratch(P, T)
                outs.append((vt.cpu().clone(), ret.cpu().clone()))
            assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1]), f"γ {gamma} λ {lam}: two runs differ"
            l32, g32 = float(np.float32(lam)), float(np.float32(gamma))
            v = _target_values(outs[0][0], ms)
            want = gr.lambda_returns(rew, done, v, l32, g32)
            S = rr.lambda_scale(rew, done, v, l32, g32)
            bar = rr.tau(T, g32, l32)
            got = outs[0][1].double().permute(2, 1, 0).numpy()
            if standardise:
                stats.update(want.reshape(-1, N), (bar * S).reshape(-1, N))
                _check_stats(a, stats, f"γ {gamma} λ {lam}")
                ratio = _standardised_ratio(got, want, S, bar, stats)
            else:
                ratio = rr.worst(got, want, S, bar)
            worst = max(worst, _record("lambda", ratio))
            assert ratio <= 1.0, f"γ {gamma} λ {lam}: a return off by {ratio:.2f} x τ S_t (τ = {bar:.2e})"
        a.close(); b.close()
    print(f"λ sweep T={T} N={N} P={P} {'standardised' if standardise else 'raw'}: worst err / (τ S_t) = {worst:.3f} "
          f"(sweep so far {WORST['lambda']:.3f})")


# ---- b. n-step returns -----------------------------------------------------------------------------------------------------------------------------
def _nstep_batch(rng, T, n, N=2, A=3):
    """envs whose episodes end at n - 1, n, n + 1 (so that t + n and t + n - 1 meet a done for t = 0, 1), at T - n, T - 1, at T, and never"""
    ends = [None, T]
    for d in (n - 1, n, n + 1, T - n, T - n + 1, T - 1):
        if 1 <= d <= T and d not in ends:
            ends.append(d)
    P = len(ends)
    s = rr.lambda_batch(rng, T, N, P, A)
    s["done"][:] = 0; s["filled"][:] = 0
    for e, end in enumerate(ends):
        s["filled"][e, : T if end is None else end] = 1
        if end is not None:
            s["done"][e, end] = 1
    s["rew"] = (rng.standard_normal(s["rew"].shape) + 0.5).astype(np.float32)
    return s, P


@pytest.mark.parametrize("T", [1, 63, 64, 65, 257])
@pytest.mark.parametrize("n", [1, 5, 63, 64])
def test_nstep_returns_where_t_plus_n_meets_T(T, n):
    N = 2
    s, P = _nstep_batch(np.random.default_rng(T * 100 + n), T, n)
    hp = lr.A2CHP(gamma=0.99, n_steps=n)
    torch.manual_seed(T + n)
    m = ac_model(hp, N, rr.D, P, T, A=3)
    m.theta_tgt.copy_(m.theta_tgt + 0.05 * torch.randn_like(m.theta_tgt))
    m.update_grads(traj_store(s, m.device), P)
    vt, ret, _ = m.scratch(P, T)
    rew, done, _ = rr.sequences(s)
    v = _target_values(vt.cpu(), None)
    g32 = float(np.float32(0.99))
    t = lambda x: torch.tensor(x, dtype=torch.float64)   # noqa: E731
    want = lr.nstep_returns(t(rew), t(done), t(v), n, g32).numpy()
    S = rr.nstep_scale(rew, done, v, n, g32)
    ratio = _record("nstep", rr.worst(ret.double().permute(2, 1, 0).cpu().numpy(), want, S, rr.nstep_tau(T, n)))
    print(f"n-step T={T} n={n} P={P}: worst err / (τ S_t) = {ratio:.3f} (sweep so far {WORST['nstep']:.3f})")
    assert ratio <= 1.0, ratio
    m.close()


# ---- c. return standardisation ---------------------------------------------------------------------------------------------------------------------
STD_SHAPES = {2: (2, 1), 255: (5, 51), 256: (16, 16), 16383: (43, 381), 16384: (64, 256), 16385: (29, 565), 32769: (99, 331), 49159: (11, 4469)}


def _std_chain(N, P, T, batches, zero_target=False):
    """three updates of one handle with standardise_returns (n-step returns, n_steps = 1): statistics and standardised returns each time"""
    hp = lr.A2CHP(gamma=0.99, n_steps=1)
    torch.manual_seed(N * 1000 + P)
    m = ac_model(hp, N, rr.D, P, T, A=3, standardise=True)
    if zero_target:   # every target value 0 in standardised units: V = the running mean, de-standardised
        m.theta_tgt.zero_()
    stats = rr.StatsRef(N)
    g32 = float(np.float32(0.99))
    worst = 0.0
    for u, make in enumerate(batches):
        ms = m.ret_ms()[:2]
        s = make(ms)
        m.update_grads(traj_store(s, m.device), P)
        vt, ret, _ = m.scratch(P, T)
        rew, done, _ = rr.sequences(s)
        v = _target_values(vt.cpu(), ms)
        t = lambda x: torch.tensor(x, dtype=torch.float64)   # noqa: E731
        want = lr.nstep_returns(t(rew), t(done), t(v), 1, g32).numpy()
        stats.update(want.reshape(-1, N))
        worst = max(worst, _check_stats(m, stats, f"N={N} P·T={P * T} update {u}"))
        S = rr.nstep_scale(rew, done, v, 1, g32)
        ratio = _standardised_ratio(ret.double().permute(2, 1, 0).cpu().numpy(), want, S, rr.nstep_tau(T, 1), stats)
        assert ratio <= 1.0, f"N={N} P·T={P * T} update {u}: a standardised return off by {ratio:.2f} x its bar"
        worst = max(worst, ratio)
    m.close()
    return worst


@pytest.mark.parametrize("N", [1, 4, 32])
@pytest.mark.parametrize("PT", list(STD_SHAPES))
def test_return_standardisation_across_the_moment_stride(PT, N):
    P, T = STD_SHAPES[PT]
    rng = np.random.default_rng(PT + N)

    def batch(ms):
        s = rr.lambda_batch(rng, T, N, P)
        s["rew"] = (rng.standard_normal(s["rew"].shape) + 0.3).astype(np.float32)
        return s

    worst = _record("standardise", _std_chain(N, P, T, [batch] * 3))
    print(f"standardisation P·T={PT} (P={P}, T={T}, {PT // rr.RET_STRIDE} full grid strides + {PT % rr.RET_STRIDE}) N={N}: worst at "
          f"{worst:.3f} of its bars")


def test_return_standardisation_of_offset_returns():
    """returns of mean ≈ 50 and spread ≈ 0.01 at P·T = 16 385: the batch variance survives only FP64 moments (tests/test_returns_edges.py)"""
    P, T, N = 29, 565, 4
    rng = np.random.default_rng(50)
    g32 = np.float32(0.99)

    def batch(ms):   # R_t = r_t + γ V_{t+1} with V the running mean: r_t = 50 + 0.01 z - γ mean, and r at T - 1 (no bootstrap) 50 + 0.01 z
        s = rr.lambda_batch(rng, T, N, P)
        s["done"][:] = 0; s["filled"][:] = 1
        r = 50.0 + 0.01 * rng.standard_normal(s["rew"].shape)
        r[:, :, : T - 1] -= (g32 * ms[0].numpy()).astype(np.float64)[None, :, None]
        s["rew"] = r.astype(np.float32)
        return s

    worst = _record("standardise", _std_chain(N, P, T, [batch] * 3, zero_target=True))
    print(f"standardisation of offset returns (mean 50, spread 0.01, P·T = {P * T}): worst at {worst:.3f} of its bars")


# ---- d. whole updates at long T ------------------------------------------------------------------------------------------------------------------
UPDATES = {
    "ia2c_mlp_indep_T257": (Case(arnn=False, crnn=False, T=257, P=8), 0.95),
    "ippo_gru_actor_T513": (Case(ppo=True, arnn=True, crnn=False, T=513, P=4, epochs=2), 1.0),
    "mappo_central_standardise_clip_T1025": (Case(ppo=True, arnn=False, crnn=False, T=1025, P=4, centralised=True, standardise=True, grad_clip=0.5,
                                                  epochs=2), 0.5),
}


@pytest.mark.parametrize("case", list(UPDATES))
@redraw_on_near_tie
def test_updates_at_long_T_match_oracle(case):
    c, lam = UPDATES[case]
    hp = _hp(c)
    m = _model(c)
    m.set_gae_lambda(lam)
    _perturb_target(m)
    st = _oracle(m, c)
    tr = Tracker(m.n_actor + m.n_critic)
    rng = np.random.default_rng(int(torch.randint(0, 1 << 30, (1,))))
    with gr.lambda_returns_in(float(np.float32(lam))):
        for u, step in enumerate(c.steps):
            s = _batch(c, rng)
            batch = ac_oracle_batch({k: v[: c.P] for k, v in s.items()})
            st0 = copy.deepcopy(st)
            want = gar.ppo_update(st, batch, hp, step, c.epochs, 0.2) if c.ppo else gar.a2c_update(st, batch, hp, step)
            if c.ppo and min(want["clip_margin"]) < TIE:
                raise NearTie(f"a ratio {min(want['clip_margin']):.1e} from the edge of the clip range")
            tgt0 = m.theta_tgt.cpu().numpy().copy()
            met = m.update_from_store(traj_store(s, m.device), c.P, step).cpu().numpy()
            _check_update(m, c, hp, st, st0, batch, want, met, step, tgt0, tr, f"{case} update {u}:")
    m.close()

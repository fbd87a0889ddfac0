"""GPU: the DQN family's TD targets per row (algorithm.td_lambda and standardise_returns; col_td_kernel, qmix_mix_kernel MODE 3, td_lambda_kernel and
ret_ms_step in csrc/dqn.cu, csrc/qmix.cuh and csrc/retms.cuh), read back through QNetwork.scratch after one update_grads, against float64.

a. td_lambda_kernel at every window and lane boundary of its split (tests/returns_ref.py TD_CASES: T mod 256 in {1, 7, 8, 9, 255, 0}, one to five
   windows, C·B mod 8 in {0, 1, 7} and C·B < 8, C·B·T on both sides of a multiple of 256, the first unfilled row, a stale restart, a done flag and a
   reward spike on the edges), IDQN, VDN and QMIX, γ in {0.99, 0.999}, λ in {0, 0.5, 0.95, 1}, raw and standardised: every row of `ret`, filled
   or not, held to |got - want| <= τ S_t against the float64 recursion over the device's own bootstrap values; each case twice, bit for bit.
b. The bootstrap values against the float64 oracle's v_{t+1}: double-Q and max, VDN's sum over agents, QMIX's target Q_tot, unstandardised with
   the statistics the update read, per row relative to the Q-values that enter it.
c. The TD head: IDQN's and VDN's dLoss/dQ equal td_dloss(float32(chosen - ret)) filled exactly, with the squared error and with the Huber loss at
   the median |δ|; the loss numerator and the filled count against their float64 sums at C·B·T = 256 k - 1, 256 k and 256 k + 1.
d. Standardisation at batch 64, 65 and 128 (VDN and QMIX keep one statistic per batch entry: ret_moments_cols_kernel above 64 entries of at most
   1024 returns each, ret_moments_kernel otherwise), T in {25, 1024, 1025}, with and without λ: the running statistics of every column against
   float64 over three updates and the standardised returns per row; and one handle moving between the two moment kernels on the same buffers.
Run with -s to see each sweep's worst err / bar."""
import types

import numpy as np
import pytest
import torch

from oracle import learner_ref as lr
from tests import qmix_options_ref as qo
from tests import returns_ref as rr
from tests import td_lambda_ref as tl
from tests.helpers import TIE, NearTie, redraw_on_near_tie, space, traj_store

pytestmark = pytest.mark.gpu
A = 6
MIXING = dict(embed_dim=32, hypernet_layers=2, hypernet_embed=32)
WORST = {}


def _record(sweep, ratio):
    WORST[sweep] = max(WORST.get(sweep, 0.0), ratio)
    return ratio


def _model(kind, N, B, T, gamma=0.99, standardise=False, double_q=True, lam=0.0, D=rr.D):
    from codebase_b200.dqn import model as M

    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=gamma, grad_clip=1.0, double_q=double_q, target_update_interval_or_tau=200.0,
                                standardise_returns=standardise, td_lambda=lam)
    args = ([space(shape=(D,))] * N, [space(n=A)] * N, cfg, [128, 128], False, False, True)
    if kind == "qmix":
        return M.QMixNetwork(*args, MIXING, "cuda", max_batch=B, max_episode_length=T)
    return (M.VDNetwork if kind == "vdn" else M.QNetwork)(*args, "cuda", max_batch=B, max_episode_length=T)


def _perturb_target(m, others=()):
    """a target that differs from the online networks; `others` get the same parameters"""
    m.theta_tgt.copy_(m.theta + 0.01 * torch.randn_like(m.theta))
    if m.mixer == 2:
        m.mix_tgt.copy_(m.mix + 0.01 * torch.randn_like(m.mix))
    m.params_changed()
    for o in others:
        for k in ("theta", "theta_tgt") + (("mix", "mix_tgt") if m.mixer == 2 else ()):
            getattr(o, k).copy_(getattr(m, k))
        o.params_changed()


def _idx(B, m):
    return torch.arange(B, dtype=torch.int32, device=m.device)


def _tm(x):
    """a device [C][B][T] buffer as time-major float64 (T, C, B)"""
    return x.detach().cpu().double().permute(2, 0, 1).numpy()


def _want(rew, done, filled, boot, lam, gamma):
    """the float64 recursion and the scale S_t over time-major (T, C, B) arrays, at float32 λ and γ"""
    l32, g32 = float(np.float32(lam)), float(np.float32(gamma))
    t = lambda x: torch.tensor(np.ascontiguousarray(x), dtype=torch.float64)   # noqa: E731
    return tl.lambda_targets(t(rew), t(done), t(filled), t(boot), l32, g32).numpy(), rr.td_lambda_scale(rew, done, filled, boot, l32, g32)


def _stat_rows(x, kind):
    """time-major (T, C, B) values as the statistics' (rows, columns): IDQN one column per agent over B·T returns, VDN and QMIX one per batch entry"""
    T, C, B = x.shape
    return x.transpose(0, 2, 1).reshape(T * B, C) if kind == "idqn" else x.reshape(T, B)


def _stat_cols(v, kind):
    """per-column statistics broadcast against (T, C, B)"""
    v = np.asarray(v, np.float64)
    return v[None, :, None] if kind == "idqn" else v[None, None, :]


def _check_stats(m, stats, what):
    mean, var, count = m.ret_ms()
    assert count == stats.count, (what, count, stats.count)
    em = np.abs(mean.double().numpy() - stats.mean) / stats.mean_bar
    ev = np.abs(var.double().numpy() - stats.var) / stats.var_bar
    assert em.max() <= 1.0 and ev.max() <= 1.0, f"{what}: running mean at {em.max():.2f}, var at {ev.max():.2f} of their bars"
    return max(float(em.max()), float(ev.max()))


def _standardised_ratio(got, want, err, stats, kind):
    """standardised returns (T, C, B) against (want - mean) / sqrt(var) of the float64 statistics: the returns' own bound err divided by the
    spread, plus the statistics' bars carried through the standardisation, plus its float32 roundings"""
    mean, var = _stat_cols(stats.mean, kind), _stat_cols(stats.var, kind)
    mbar, vbar = _stat_cols(stats.mean_bar, kind), _stat_cols(stats.var_bar, kind)
    sd = np.sqrt(var)
    z = (want - mean) / sd
    zbar = (err + mbar) / sd + (0.5 * vbar / var + 4 * rr.U32) * np.abs(z)
    return float((np.abs(got - z) / zbar).max())


# ---- a. the scan at every boundary of its split ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("standardise", [False, True], ids=["raw", "standardise"])
@pytest.mark.parametrize("T,kind,N,cb8,cbt", rr.TD_CASES)
def test_td_lambda_targets_at_the_split_boundaries(T, kind, N, cb8, cbt, standardise):
    C, B = rr.td_case(T, kind, N, cb8, cbt)
    s = rr.td_batch(np.random.default_rng(T * 7 + N), T, N, B)
    rew, done, filled = rr.td_sequences(s, C)
    worst = 0.0
    for gamma in rr.GAMMAS:
        torch.manual_seed(T * 31 + N)
        a, b = (_model(kind, N, B, T, gamma, standardise) for _ in range(2))
        _perturb_target(a, [b])
        ts, idx = traj_store(s, a.device), _idx(B, a)
        stats = rr.StatsRef(C if kind == "idqn" else B) if standardise else None
        for lam in rr.LAMBDAS:
            outs = []
            for m in (a, b):
                m.set_td_lambda(lam)
                m.update_grads(ts, idx)
                boot, ret, _, _ = m.scratch(B, T)
                outs.append((boot.cpu().clone(), ret.cpu().clone()))
            assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1]), f"γ {gamma} λ {lam}: two runs differ"
            want, S = _want(rew, done, filled, _tm(outs[0][0]), lam, gamma)
            bar = rr.td_tau(T, gamma, lam)
            got = _tm(outs[0][1])
            if standardise:
                stats.update(_stat_rows(want, kind), _stat_rows(bar * S, kind))
                _check_stats(a, stats, f"γ {gamma} λ {lam}")
                ratio = _standardised_ratio(got, want, bar * S, stats, kind)
            else:
                ratio = rr.worst(got, want, S, bar)
            worst = max(worst, _record("scan", ratio))
            assert ratio <= 1.0, f"γ {gamma} λ {lam}: a target off by {ratio:.2f} x τ S_t (τ = {bar:.2e})"
        a.close(); b.close()
    print(f"scan T={T} {kind} C={C} B={B} {'standardised' if standardise else 'raw'} (ret_ms {rr.ret_ms_path(kind, N, B, T)}): worst err / bar = "
          f"{worst:.3f} (sweep so far {WORST['scan']:.3f})")


# ---- b. the bootstrap values ---------------------------------------------------------------------------------------------------------------------
def _oracle_boot(m, kind, s, double_q, ms):
    """the float64 oracle's v_{t+1} as [C][B][T], de-standardised with ms = (mean, var) (or None), and each row's scale: the |Q| that enter it"""
    N, D = m.n_agents, m.in_dim
    batch = lr.batch_from_store(s, np.arange(s["filled"].shape[0]))
    obss = batch["obss"].double()
    with torch.no_grad():
        q = torch.stack(lr.agents_forward(m.theta.cpu().double(), m.agent_net, list(obss), D, A))[:, 1:]       # (N, T, B, A)
        tq = torch.stack(lr.agents_forward(m.theta_tgt.cpu().double(), m.agent_net, list(obss), D, A))[:, 1:]
    if double_q:
        top2 = q.topk(2, dim=-1).values
        gap = float(((top2[..., 0] - top2[..., 1]) / top2[..., 0].abs().clamp_min(1.0)).min())
        if gap < TIE:
            raise NearTie(f"double-Q argmax margin {gap:.1e} on some row")
        v = tq.gather(-1, q.argmax(-1, keepdim=True)).squeeze(-1)                                               # (N, T, B)
    else:
        v = tq.max(-1)[0]
    mag = tq.abs().max(-1)[0]
    if kind == "idqn":
        v, mag = v.permute(0, 2, 1), mag.permute(0, 2, 1)
    elif kind == "vdn":
        v, mag = v.sum(0).T[None], mag.sum(0).T[None]
    else:
        states = torch.concat(list(obss[:, 1:]), dim=-1)
        v = qo.mixer_forward(m.mix_tgt.cpu().double(), v, states, N, m.embed_dim, m.hypernet_embed, m.hypernet_layers)     # (T, B)
        v, mag = v.T[None], (mag.sum(0).T + v.abs().T)[None]
    v, mag = v.numpy(), mag.numpy() + 1.0
    if ms is not None:
        mean, var = (x.double().numpy() for x in ms)
        cols = (lambda x: x[:, None, None]) if kind == "idqn" else (lambda x: x[None, :, None])
        v = v * np.sqrt(cols(var)) + cols(mean)
        mag = mag * np.sqrt(cols(var)) + np.abs(cols(mean))
    return v, mag


BOOT_BAR = 2e-5   # the float32 forward passes (3xTF32 agents, FP32 mixer) agree with float64 to ~1e-6 of the Q-values that enter the row
BOOT = {"idqn_double_q": ("idqn", True, False, 25, 8), "idqn_max_standardise": ("idqn", False, True, 257, 4),
        "vdn_double_q": ("vdn", True, False, 25, 8), "vdn_max_standardise": ("vdn", False, True, 9, 16),
        "qmix_double_q": ("qmix", True, False, 25, 8), "qmix_max_standardise": ("qmix", False, True, 25, 8)}


@pytest.mark.parametrize("name", list(BOOT))
@redraw_on_near_tie
def test_bootstrap_values_match_the_oracle(name):
    kind, double_q, standardise, T, B = BOOT[name]
    N = 2
    m = _model(kind, N, B, T, standardise=standardise, double_q=double_q, lam=0.5)
    _perturb_target(m)
    worst = 0.0
    for u in range(2):   # the second update reads the statistics the first one left
        s = rr.td_batch(np.random.default_rng(100 * u + T), T, N, B)
        ms = m.ret_ms()[:2] if standardise else None
        want, mag = _oracle_boot(m, kind, s, double_q, ms)
        m.update_grads(traj_store(s, m.device), _idx(B, m))
        got = m.scratch(B, T)[0].cpu().double().numpy()
        ratio = float((np.abs(got - want) / (BOOT_BAR * mag)).max())
        worst = max(worst, _record("boot", ratio))
        assert ratio <= 1.0, f"{name} update {u}: a bootstrap value off by {ratio:.2f} x its bar"
    print(f"bootstrap {name}: worst err / bar = {worst:.3f}")
    m.close()


# ---- c. the TD head ------------------------------------------------------------------------------------------------------------------------------
def _dloss(d, huber):
    return np.clip(d, np.float32(-huber), np.float32(huber)) if huber else np.float32(2.0) * d


def _loss64(d, huber):
    ad = np.abs(d)
    return np.where(ad < huber, 0.5 * d * d, huber * (ad - 0.5 * huber)) if huber else d * d


# (kind, N, T, B): C·B·T = 513, 1023, 512, 511, 512, 513
HEAD = [("idqn", 3, 9, 19), ("idqn", 3, 11, 31), ("idqn", 2, 16, 16), ("vdn", 2, 7, 73), ("vdn", 2, 16, 32), ("vdn", 2, 27, 19)]


@pytest.mark.parametrize("kind,N,T,B", HEAD)
def test_td_head_is_the_rule_on_the_targets(kind, N, T, B):
    C = rr.td_columns(kind, N)
    torch.manual_seed(T * B)
    m = _model(kind, N, B, T, double_q=False, lam=0.8)
    _perturb_target(m)
    s = rr.td_batch(np.random.default_rng(T * B), T, N, B)
    ts, idx = traj_store(s, m.device), _idx(B, m)
    fill = np.broadcast_to(s["filled"].astype(np.float32)[None], (C, B, T))
    huber = None
    for pass_ in ("squared", "huber"):
        if pass_ == "huber":
            huber = float(np.float32(np.median(np.abs(d64[fill > 0]))))
            m.set_huber_delta(huber)
        m.update_grads(ts, idx)
        _, ret, chosen, td = (x.cpu().numpy() for x in m.scratch(B, T))
        d = (chosen - ret).astype(np.float32)
        want = _dloss(d, huber) * fill
        assert np.array_equal(td, want), f"{pass_}: dLoss/dQ differs from the rule at {np.count_nonzero(td != want)} rows"
        d64 = chosen.astype(np.float64) - ret.astype(np.float64)
        num = float((_loss64(d64, huber) * fill).sum())
        g = m.grad[m.n_params: m.n_params + 2].cpu().double().numpy()
        assert g[1] == float(s["filled"].sum()), (pass_, g[1], s["filled"].sum())
        assert abs(g[0] - num) <= 1e-5 * num, f"{pass_}: loss numerator {g[0]} vs {num} at C·B·T = {C * B * T}"
        print(f"TD head {kind} C·B·T={C * B * T} {pass_}: exact; loss numerator off by {abs(g[0] - num) / num:.1e} relative")
    m.close()


# ---- d. standardisation at batch sizes above 64 -----------------------------------------------------------------------------------------------
def _targets(m, kind, s, lam, ms):
    """(want (T, 1, B), per-row bound) of the update about to run: with λ, the recursion over the device's bootstrap values (read after it, see
    the caller); without, the one-step target over the oracle's v"""
    v, mag = _oracle_boot(m, kind, s, False, ms)
    rew, done, filled = rr.td_sequences(s, 1)
    g32 = float(np.float32(m.gamma))
    vt = v.transpose(2, 0, 1)
    want = rew + g32 * (1.0 - done[1:]) * vt
    err = g32 * BOOT_BAR * mag.transpose(2, 0, 1) + 4 * rr.U32 * (np.abs(rew) + g32 * np.abs(vt))
    return want, err


def _std_update(m, kind, s, lam, stats, what):
    """one standardised update of a VDN / QMIX handle on store s: statistics and standardised returns against float64"""
    B, T = s["filled"].shape
    ms = m.ret_ms()[:2]
    if lam is None:
        want, err = _targets(m, kind, s, lam, ms)
    m.update_grads(traj_store(s, m.device), _idx(B, m))
    boot, ret, _, _ = m.scratch(B, T)
    if lam is not None:
        rew, done, filled = rr.td_sequences(s, 1)
        want, S = _want(rew, done, filled, _tm(boot), lam, m.gamma)
        err = rr.td_tau(T, m.gamma, lam) * S
    stats.update(_stat_rows(want, kind), _stat_rows(err, kind))
    r1 = _check_stats(m, stats, what)
    r2 = _standardised_ratio(_tm(ret), want, err, stats, kind)
    assert r2 <= 1.0, f"{what}: a standardised target off by {r2:.2f} x its bar"
    return max(r1, r2)


@pytest.mark.parametrize("lam", [None, 0.95], ids=["one_step", "lambda"])
@pytest.mark.parametrize("T", [25, 1024, 1025])
@pytest.mark.parametrize("B", [64, 65, 128])
@pytest.mark.parametrize("kind", ["vdn", "qmix"])
def test_standardisation_above_64_batch_entries(kind, B, T, lam):
    N = 2
    torch.manual_seed(B + T)
    m = _model(kind, N, B, T, standardise=True, double_q=False, lam=lam)
    _perturb_target(m)
    stats = rr.StatsRef(B)
    rng = np.random.default_rng(B * T)
    worst = 0.0
    for u in range(3):
        worst = max(worst, _std_update(m, kind, rr.td_batch(rng, T, N, B), lam, stats, f"update {u}"))
    _record("standardise", worst)
    print(f"standardisation {kind} B={B} T={T} λ={lam} (ret_ms {rr.ret_ms_path(kind, N, B, T)}): worst at {worst:.3f} of its bars")
    m.close()


@pytest.mark.parametrize("kind", ["vdn", "qmix"])
def test_one_handle_moves_between_the_moment_kernels(kind):
    """B = 65 at T = 1025 (ret_moments_kernel: every block's partials), 25 (ret_moments_cols_kernel: block 0's, the others zeroed), 1025"""
    N, B = 2, 65
    torch.manual_seed(65)
    m = _model(kind, N, B, 1025, standardise=True, double_q=False, lam=0.95)
    _perturb_target(m)
    stats = rr.StatsRef(B)
    rng = np.random.default_rng(1025)
    worst = 0.0
    for u, T in enumerate((1025, 25, 1025)):
        assert rr.ret_ms_path(kind, N, B, T) == ("cols" if T == 25 else "grid")
        worst = max(worst, _std_update(m, kind, rr.td_batch(rng, T, N, B), 0.95, stats, f"update {u} at T = {T}"))
    _record("standardise", worst)
    print(f"{kind} B=65 at T = 1025, 25, 1025: worst at {worst:.3f} of its bars")
    m.close()

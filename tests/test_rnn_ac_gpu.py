"""GPU: recurrent (GRU) actor and critic networks of IA2C / IPPO / MAA2C / MAPPO (csrc/gru_kernels.cu behind marl_a2c_create_rnn) against the oracle
restatement (tests/gru_ac_ref.py, itself pinned to the reference's outputs by test_rnn_ac.py): the act step carrying h for actor, critic and target
critic, single updates on ragged batches (every epoch's gradient for PPO), the goldens, update chains that are never re-synchronised with the oracle,
bit-for-bit determinism, and the training driver end to end."""
import copy
import ctypes as C
import dataclasses
import types

import numpy as np
import pytest
import torch

from oracle import learner_ref as lr
from tests import gru_ac_ref as gar
from tests.helpers import TIE, NearTie, ac_batch, ac_oracle_batch, assert_grad_close, clipped, close_scaled, redraw_on_near_tie, space, traj_store

pytestmark = pytest.mark.gpu
GRU_NAMES = ("W1", "b1", "W_ih", "W_hh", "b_ih", "b_hh", "W3", "b3")


@dataclasses.dataclass(frozen=True)
class Case:
    ppo: bool = False
    arnn: bool = True            # actor.use_rnn
    crnn: bool = True            # critic.use_rnn
    N: int = 2
    D: int = 15
    A: int = 6
    sharing: object = False
    centralised: bool = False
    P: int = 32                  # environments of each update (n_envs)
    cap: int = 0                 # store capacity and max_envs (0: P)
    T: int = 7
    steps: tuple = (0,)          # environment step of each update (hard syncs where step % tu == 0)
    tu: float = 200
    grad_clip: float = 0.0
    lr: float = 3e-4
    n_steps: int = 5
    epochs: int = 4
    standardise: bool = False
    clip_reached: bool = False   # PPO: the oracle's surrogate must block some entries' gradient in some update


def _hp(c):
    return lr.A2CHP(lr=c.lr, gamma=0.99, grad_clip=c.grad_clip, n_steps=c.n_steps, entropy_coef=0.001, value_loss_coef=0.5, target_update_interval_or_tau=c.tu)


def _model(c):
    from codebase_b200.ac import model as M

    hp = _hp(c)
    sharing = list(c.sharing) if isinstance(c.sharing, tuple) else c.sharing
    cfg = types.SimpleNamespace(optimizer="Adam", lr=hp.lr, gamma=hp.gamma, grad_clip=hp.grad_clip, n_steps=hp.n_steps, entropy_coef=hp.entropy_coef,
                                value_loss_coef=hp.value_loss_coef, target_update_interval_or_tau=hp.target_update_interval_or_tau,
                                standardise_returns=c.standardise, num_epochs=c.epochs, ppo_clip=0.2)
    anet = types.SimpleNamespace(layers=[128, 128], parameter_sharing=sharing, use_rnn=c.arnn, use_orthogonal_init=True, centralised=False)
    cnet = types.SimpleNamespace(layers=[128, 128], parameter_sharing=sharing, use_rnn=c.crnn, use_orthogonal_init=True, centralised=c.centralised)
    return (M.PPONetwork if c.ppo else M.A2CNetwork)([space(shape=(c.D,))] * c.N, [space(n=c.A)] * c.N, cfg, anet, cnet, "cuda",
                                                    max_envs=c.cap or c.P, max_episode_length=c.T)


def _oracle(m, c):
    return lr.A2CState(m.theta[: m.n_actor].cpu().clone(), m.theta[m.n_actor:].cpu().clone(), m.theta_tgt.cpu().clone(), list(m.actor_net),
                       list(m.critic_net), c.D, c.A, centralised=c.centralised, ret_ms=lr.RunningMeanStdRef((c.N,)) if c.standardise else None)


def _perturb_target(m):
    """a target critic that differs from the critic until the first sync, so that the target's values and update rule matter"""
    m.theta_tgt.copy_(m.theta_tgt + 0.01 * torch.randn_like(m.theta_tgt))


def _batch(c, rng):
    s = ac_batch(rng, c.cap or c.P, c.N, c.T, c.D, A=c.A)
    s["obs"] = (s["obs"] / 6.0).astype(np.float32)   # LBF-like magnitudes keep the GRU away from saturation
    return s


def _blocks(m, c):
    """(name, slice) of every tensor of every actor and critic network in the flat [actor | critic] vector, GRU or MLP, at the model's widths"""
    out, o = [], 0
    for part, rnn, n_nets, shapes in (("actor", c.arnn, m.n_actor_nets, m._actor_shapes), ("critic", c.crnn, m.n_critic_nets, m._critic_shapes)):
        names = GRU_NAMES if rnn else ("W1", "b1", "W2", "b2", "W3", "b3")
        assert len(names) == len(shapes), (part, shapes)
        for k in range(n_nets):
            for name, (_, shape) in zip(names, shapes):
                size = int(np.prod(shape))
                out.append((f"{part}{k}.{name}", slice(o, o + size)))
                o += size
    assert o == m.n_actor + m.n_critic
    return out


def _close(a, b, tol, what):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert np.allclose(a, b, rtol=tol, atol=tol), (what, float(np.abs(a - b).max()))


def _polyak_close(got, old, new, tau):
    """got == (1 - tau) old + tau new in float32, to 1 ulp of any of the three roundings (plain, or contracted to an FMA either way)"""
    t = np.float32(tau)
    a = np.float32(1) - t
    plain = (a * old + t * new).astype(np.float32)
    fma1 = (a.astype(np.float64) * old + (t * new).astype(np.float64)).astype(np.float32)
    fma2 = (t.astype(np.float64) * new + (a * old).astype(np.float64)).astype(np.float32)
    err = np.min([np.abs(got.astype(np.float64) - x) / np.spacing(np.abs(x)) for x in (plain, fma1, fma2)], axis=0)
    assert err.max() <= 1.0, f"Polyak target off by {err.max():.1f} ulp"


class Tracker:
    """what the per-update checks carry across the updates of a chain: elements whose oracle gradient was ill-conditioned on some optimiser step,
    and Adam's m without cancellation (the same moving average of |clipped gradient|) as m's scale"""

    def __init__(self, n):
        self.excused, self.abs_m, self.clip_seen, self.updates = np.zeros(n, bool), np.zeros(n), False, 0


def _oracle_update(c, st, batch, hp, step):
    want = gar.ppo_update(st, batch, hp, step, c.epochs, 0.2) if c.ppo else gar.a2c_update(st, batch, hp, step)
    if c.ppo and min(want["clip_margin"]) < TIE:   # a ratio on the edge of the clip range: the surrogate's gradient jumps there
        raise NearTie(f"a ratio {min(want['clip_margin']):.1e} from the edge of the clip range")
    return want


def _check_update(m, c, hp, st, st0, batch, want, met, step, tgt0, tr, what, tol=2e-5):
    """every per-update check of test_ac_chain_gpu.py: returns, target values, advantages, raw and clipped gradients, metrics, Adam m / v per tensor,
    parameters element by element (except where Adam is ill-conditioned), the target critic's own rule, the running return statistics"""
    n, na = m.n_actor + m.n_critic, m.n_actor
    tr.updates += 1
    vt, ret, adv = (x.cpu().numpy() for x in m.scratch(c.P, c.T))
    _close(ret, want["returns"].permute(2, 1, 0).numpy(), tol, f"{what} returns")
    _close(vt, want["next_value"].permute(2, 1, 0).numpy(), 1e-5, f"{what} target values")
    if c.ppo:
        tr.clip_seen |= max(want["clip_frac"]) > 0
        raws = [np.concatenate([g["actor"].numpy(), g["critic"].numpy()]) for g in want["grads"]]
        steps_clipped = [np.concatenate([g["actor"].numpy(), g["critic"].numpy()]) for g in want["grads_clipped"]]
        want_norm = float(np.mean(want["grad_norms"]))
        risk = lambda: gar.ppo_kink_risk(st0, batch, hp, want, 0.2)   # noqa: E731 -- the last epoch's loss, at the parameters it started from
    else:
        _close(adv, want["advantages"].permute(2, 1, 0).numpy(), tol, f"{what} advantages")
        raws = [np.concatenate([want["grad"]["actor"].numpy(), want["grad"]["critic"].numpy()])]
        steps_clipped = [np.concatenate([want["grad_clipped"]["actor"].numpy(), want["grad_clipped"]["critic"].numpy()])]
        want_norm = want["grad_norm"]
        risk = lambda: gar.a2c_kink_risk(st0, batch, hp)   # noqa: E731
    g = m.grad.cpu().numpy()
    fill = float(batch["filled"].sum())
    assert g[n + 1] == fill and met[4] == fill, (what, g[n + 1], met[4], fill)
    assert_grad_close(lr, st0, batch, hp, g[:n] / fill, raws[-1], tol=tol, what=what, kink_risk=risk)
    close_scaled(clipped(g[:n] / fill, c.grad_clip), steps_clipped[-1], tol)
    got = m.metrics_dict(torch.tensor(met))
    _close([got[k] for k in ("loss", "actor_loss", "value_loss", "entropy")], [want[k] for k in ("loss", "actor_loss", "value_loss", "entropy")], tol, what)
    assert np.allclose(met[1], want_norm, rtol=1e-4, atol=1e-5), (what, met[1], want_norm)
    blocks = _blocks(m, c)
    for gc in steps_clipped:
        tr.abs_m += (np.abs(gc) - tr.abs_m) * (1 - 0.9)
    wm = np.concatenate([st.m["actor"].numpy(), st.m["critic"].numpy()]); wv = np.concatenate([st.v["actor"].numpy(), st.v["critic"].numpy()])
    am, av = m.adam_m.cpu().numpy(), m.adam_v.cpu().numpy()
    for name, sl in blocks:
        err = np.abs(am[sl].astype(np.float64) - wm[sl]).max()
        assert err <= 2 * tol * tr.abs_m[sl].max() + 1e-30, f"{what} Adam m of {name}: {err:.3e} > {2 * tol:g} x {tr.abs_m[sl].max():.3e}"
        try:
            close_scaled(av[sl], wv[sl], 4 * tol)
        except AssertionError as e:
            raise AssertionError(f"{what} Adam v of {name}: {e}") from None
    for r in raws:
        for name, sl in blocks:
            low = np.abs(r[sl]) < 1e-4 * np.abs(r[sl]).max()
            if name.endswith("b3") and low.any():   # the oracle's own gradient, not the device's: an unlucky draw, re-drawn, never excused
                raise NearTie(f"{what} the oracle's gradient of {name} is below 1e-4 of the block's largest")
            tr.excused[sl] |= low
    th, want_th = m.theta.cpu().numpy(), np.concatenate([st.actor.numpy(), st.critic.numpy()])
    tg = m.theta_tgt.cpu().numpy()
    for name, mine, theirs, exc in (("theta", th, want_th, tr.excused), ("target", tg, st.target.numpy(), tr.excused[na:])):
        d = np.abs(mine - theirs)
        assert d.max() < 2 * c.lr * (c.epochs if c.ppo else 1) * tr.updates + 1e-6, (what, name, d.max())   # an excused element still moves like Adam
        bad = np.flatnonzero((d > tol * max(1.0, c.lr / 3e-4)) & ~exc)
        assert bad.size == 0, f"{what} {name}: {bad.size} elements off by up to {d[bad].max():.2e} (first {bad[:5]})"
    critic = th[na:]
    if c.tu > 1 and step % c.tu == 0:
        assert np.array_equal(tg, critic), f"{what} the hard sync must copy the critic bit for bit"
    elif c.tu > 1:
        assert np.array_equal(tg, tgt0), f"{what} the target changed without a sync"
    else:
        _polyak_close(tg, tgt0, critic, c.tu)
    if c.standardise:
        mean, var, count = m.ret_ms()
        _close(mean.numpy(), st.ret_ms.mean.numpy(), 1e-5, f"{what} running mean"); _close(var.numpy(), st.ret_ms.var.numpy(), 1e-5, f"{what} running var")
        assert abs(count - st.ret_ms.count) < 1e-6, (what, count, st.ret_ms.count)


# ---- 1. the act step ----------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sharing,central,N,D,A", [(False, False, 2, 15, 6), (True, True, 2, 15, 8), ([0, 0, 1], False, 3, 11, 3), (False, True, 2, 16, 6)])
def test_act_steps_carry_h_like_the_oracle(sharing, central, N, D, A):
    """ten carried steps of marl_a2c_forward_rnn for the actor, the critic and the target critic against the oracle's recurrence (outputs and h at
    every step); h_in = NULL equals explicit zeros bit for bit; aliasing h_in / h_out and calls on the wrong part are refused"""
    from codebase_b200 import _native as nat

    c = Case(N=N, D=D, A=A, sharing=tuple(sharing) if isinstance(sharing, list) else sharing, centralised=central, P=8, T=4)
    torch.manual_seed(D * 10 + A)
    m = _model(c)
    _perturb_target(m)
    E, S = 37, 10
    obs = (torch.randint(-1, 12, (S, E, N, D)) / 6.0).float()
    cobs = gar.joint(obs) if central else obs
    want_l, want_lh = gar.act_steps(m.theta[: m.n_actor].cpu(), list(m.actor_net), obs, D, A)
    want_v, want_vh = gar.act_steps(m.theta[m.n_actor:].cpu(), list(m.critic_net), cobs, m.critic_in, 1)
    want_t, want_th = gar.act_steps(m.theta_tgt.cpu(), list(m.critic_net), cobs, m.critic_in, 1)
    ha = hv = ht = None
    for s in range(S):
        o = obs[s].cuda().contiguous()
        lg, ha_new = m.logits(o, h=ha)
        v, hv_new = m.values(o, h=hv)
        t, ht_new = m.values(o, target=True, h=ht)
        for got, want, what in ((lg, want_l[s], "logits"), (ha_new, want_lh[s], "actor h"), (v, want_v[s, ..., 0], "values"), (hv_new, want_vh[s], "critic h"),
                                (t, want_t[s, ..., 0], "target values"), (ht_new, want_th[s], "target h")):
            np.testing.assert_allclose(got.cpu().numpy(), want.numpy(), rtol=0, atol=1e-5 * max(1.0, float(want.abs().max())), err_msg=f"{what} step {s}")
        ha, hv, ht = ha_new.clone(), hv_new.clone(), ht_new.clone()
    o = obs[0].cuda().contiguous()
    for fwd in (lambda h: m.logits(o, h=h), lambda h: m.values(o, h=h), lambda h: m.values(o, target=True, h=h)):
        a0, h0 = fwd(None)
        a1, h1 = fwd(torch.zeros(E, N, 128, device="cuda"))
        assert torch.equal(a0, a1) and torch.equal(h0, h1)
    with pytest.raises(nat.NativeError, match="alias"):
        m.logits(o, h=ha, h_out=ha)
    out = torch.empty(E, N, A, device="cuda")
    with pytest.raises(nat.NativeError, match="marl_a2c_forward_rnn"):
        nat.check(m._lib.marl_a2c_forward_actor(m._h, nat.ptr(o), C.c_int32(E), nat.ptr(out), nat.stream_ptr()), "marl_a2c_forward_actor")
    with pytest.raises(nat.NativeError, match="marl_a2c_forward_rnn"):
        nat.check(m._lib.marl_a2c_forward_critic(m._h, nat.ptr(o), C.c_int32(E), C.c_int32(0), nat.ptr(out), nat.stream_ptr()), "marl_a2c_forward_critic")
    m.close()
    # a part that is not recurrent is refused by marl_a2c_forward_rnn
    mixed = _model(dataclasses.replace(c, crnn=False))
    with pytest.raises(nat.NativeError, match="not recurrent"):
        nat.check(mixed._lib.marl_a2c_forward_rnn(mixed._h, C.c_int32(1), nat.ptr(o), C.c_int32(E), None, None, nat.ptr(out), nat.stream_ptr()), "marl_a2c_forward_rnn")
    mixed.close()


# ---- 2. single updates against the oracle ------------------------------------------------------------------------------------------------------
ONE = {
    "ia2c_T1_N1_A3": Case(T=1, N=1, A=3, P=24),
    "ia2c_T7_shared_A8_below_max_envs": Case(T=7, sharing=True, A=8, P=40, cap=56),
    "ia2c_T25_N4_seps_clip": Case(T=25, N=4, sharing=(0, 1, 1, 0), D=7, P=20, grad_clip=0.5),
    "maa2c_T7_central": Case(T=7, centralised=True, P=32),
    "ia2c_T7_standardise": Case(T=7, standardise=True, P=32),
    "ia2c_rnn_actor_mlp_critic": Case(T=7, crnn=False, P=32),
    "maa2c_mlp_actor_rnn_central_critic": Case(T=7, arnn=False, centralised=True, P=32),
    "ippo_T10_clip_reached": Case(ppo=True, T=10, P=16, lr=3e-3, epochs=6, grad_clip=0.5, tu=0.05, clip_reached=True),
    "mappo_T25_shared": Case(ppo=True, T=25, P=24, sharing=True, centralised=True, epochs=2),
}


@pytest.mark.parametrize("case", list(ONE))
@redraw_on_near_tie
def test_single_update_matches_oracle(case):
    """one update (hard sync at step 0): target values, returns, advantages, raw and clipped gradient, metrics, Adam m / v, parameters, target.
    PPO: every epoch's raw gradient, from handles that stop after 1, 2, ... epochs (the first epoch's ratio is 1 only with the right old
    log-probabilities)"""
    c = ONE[case]
    hp = _hp(c)
    m = _model(c)
    _perturb_target(m)
    st = _oracle(m, c)
    th0, tgt0 = m.theta.detach().clone(), m.theta_tgt.detach().clone()
    s = _batch(c, np.random.default_rng(int(torch.randint(0, 1 << 30, (1,)))))
    batch = ac_oracle_batch({k: v[: c.P] for k, v in s.items()})
    st0 = copy.deepcopy(st)
    want = _oracle_update(c, st, batch, hp, 0)
    ts = traj_store(s, m.device)
    met = m.update_from_store(ts, c.P, 0).cpu().numpy()
    tr = Tracker(m.n_actor + m.n_critic)
    _check_update(m, c, hp, st, st0, batch, want, met, 0, tgt0.cpu().numpy(), tr, case)
    if c.ppo:
        n, fill = m.n_actor + m.n_critic, float(batch["filled"].sum())
        for e in range(1, c.epochs + 1):
            m2 = _model(c)
            m2.theta.copy_(th0); m2.theta_tgt.copy_(tgt0)
            m2.num_epochs = e
            m2.update_from_store(ts, c.P, 0)
            raw = np.concatenate([want["grads"][e - 1]["actor"].numpy(), want["grads"][e - 1]["critic"].numpy()])
            assert_grad_close(lr, st0, batch, hp, m2.grad.cpu().numpy()[:n] / fill, raw, tol=2e-5, what=f"{case} epoch {e}",
                              kink_risk=lambda: gar.ppo_kink_risk(st0, batch, hp, want, 0.2, e - 1))
            m2.close()
        if c.clip_reached:
            assert tr.clip_seen, "the clipped surrogate was never reached"
    m.close()


# ---- 3. the goldens (the reference's own numbers) ------------------------------------------------------------------------------------------------
def _golden_case(name):
    import tests.test_rnn_ac as cpu

    ppo, arnn, crnn, sharing, central, D, kw, standardise, _ = cpu.CASES[name]
    hp = cpu.case_setup(name)[0]
    return Case(ppo=ppo, arnn=arnn, crnn=crnn, N=cpu.N, D=D, A=cpu.A, sharing=sharing, centralised=central, P=cpu.P, T=cpu.T,
                tu=hp.target_update_interval_or_tau, grad_clip=hp.grad_clip, lr=hp.lr, epochs=cpu.EPOCHS, standardise=standardise)


@pytest.mark.parametrize("name", ["ia2c_indep", "ia2c_shared_clip_polyak", "ippo_indep_clip", "mappo_shared_central", "ia2c_standardise",
                                  "ia2c_rnn_actor_mlp_critic"])
def test_fixture_updates_match_reference_golden(name):
    import tests.test_rnn_ac as cpu

    g = np.load(cpu.golden_path(name))
    c = _golden_case(name)
    _, D, CD, nets, actor0, critic0, _, _ = cpu.case_setup(name)
    m = _model(c)
    m.theta.copy_(torch.cat([actor0, critic0])); m.theta_tgt.copy_(critic0)
    n = m.n_actor + m.n_critic
    for u, step in enumerate(cpu.STEPS):
        s = {k: g[f"b{u}_{k}"] for k in ("obs", "act", "rew", "done", "filled")}
        met = m.update_from_store(traj_store(s, m.device), c.P, step).cpu()
        got = m.metrics_dict(met)
        np.testing.assert_allclose([got[k] for k in ("loss", "actor_loss", "value_loss", "entropy")], g["metrics"][u], rtol=2e-5, atol=2e-5, err_msg=f"update {u}")
        if u == 0:
            gr_ = m.grad.cpu().numpy()
            gc = clipped(gr_[:n] / gr_[n + 1], c.grad_clip)[:: cpu.STRIDE]
            assert np.abs(gc - g["grad0"]).max() <= 2e-5 * max(1.0, float(np.abs(g["grad0"]).max()))
    th = m.theta.cpu().numpy()
    for got, key in ((th[: m.n_actor], "actor3"), (th[m.n_actor:], "critic3"), (m.theta_tgt.cpu().numpy(), "target3")):
        d = np.abs(got[:: cpu.STRIDE] - g[key])
        assert np.quantile(d, 0.999) < 1e-5 * max(1.0, c.lr / 3e-4) and d.max() < 2 * c.lr * 3 * (c.epochs if c.ppo else 1), key
    cut = len(range(0, m.n_actor, cpu.STRIDE))
    for key, got, tol in (("m3", m.adam_m.cpu().numpy()[:: cpu.STRIDE], 5e-5), ("v3", m.adam_v.cpu().numpy()[:: cpu.STRIDE], 1e-4)):
        for sl in (slice(0, cut), slice(cut, None)):
            close_scaled(got[sl], g[key][sl], tol)
    if c.standardise:
        mean, var, count = m.ret_ms()
        np.testing.assert_allclose(mean.numpy(), g["ret_mean"], rtol=1e-5, atol=1e-6); np.testing.assert_allclose(var.numpy(), g["ret_var"], rtol=1e-5)
    m.close()
    m = _model(c)   # the act steps were recorded at the initial parameters
    m.theta.copy_(torch.cat([actor0, critic0])); m.theta_tgt.copy_(critic0)
    ha = hv = None
    for s in range(10):
        o = torch.tensor(g["act_obs"][s]).view(1, c.N, c.D).cuda()
        if c.arnn:
            lg, ha = m.logits(o, h=ha)
            np.testing.assert_allclose(ha[0].cpu().numpy(), g["act_h"][s], rtol=0, atol=1e-5)
            ha = ha.clone()
        else:
            lg = m.logits(o)
        np.testing.assert_allclose(lg[0].cpu().numpy(), g["act_logits"][s], rtol=0, atol=1e-5)
        if c.crnn:
            v, hv = m.values(o, h=hv)
            np.testing.assert_allclose(hv[0].cpu().numpy(), g["value_h"][s], rtol=0, atol=1e-5)
            hv = hv.clone()
        else:
            v = m.values(o)
        np.testing.assert_allclose(v[0].cpu().numpy(), g["act_values"][s], rtol=0, atol=1e-5)
    m.close()


# ---- 4. unglued chains -------------------------------------------------------------------------------------------------------------------------
CHAIN = {
    "ia2c_hard": Case(T=25, P=48, tu=200, steps=(0, 64, 128, 200, 264, 400, 464, 600)),
    "ia2c_shared_polyak_clip": Case(T=25, P=48, sharing=True, tu=0.05, grad_clip=0.5, steps=tuple(range(8))),
    "ippo_hard": Case(ppo=True, T=10, P=32, tu=2, steps=(0, 3, 4, 5, 6, 7, 8, 9)),
    "ippo_polyak_rnn_actor_mlp_critic": Case(ppo=True, crnn=False, T=10, P=32, tu=0.05, steps=tuple(range(8))),
    "mappo_hard_standardise": Case(ppo=True, centralised=True, standardise=True, sharing=True, T=10, P=32, tu=2, epochs=2, steps=(0, 3, 4, 5, 6, 7, 8, 9)),
}


def _chain_batches(c):
    rng = np.random.default_rng(c.P * 7 + c.T * 3 + c.A)
    return [_batch(c, rng) for _ in c.steps]


@pytest.mark.parametrize("case", list(CHAIN))
@redraw_on_near_tie
def test_chain_matches_oracle(case):
    """eight or more updates that are never re-synchronised with the oracle: the device carries parameters, Adam and its step counter, the target
    critic and the return statistics on its own; after every update the checks of test_ac_chain_gpu.py"""
    c = CHAIN[case]
    hp = _hp(c)
    m = _model(c)
    _perturb_target(m)
    st = _oracle(m, c)
    tr = Tracker(m.n_actor + m.n_critic)
    for u, (step, s) in enumerate(zip(c.steps, _chain_batches(c))):
        batch = ac_oracle_batch({k: v[: c.P] for k, v in s.items()})
        st0 = copy.deepcopy(st)
        want = _oracle_update(c, st, batch, hp, step)
        tgt0 = m.theta_tgt.cpu().numpy().copy()
        met = m.update_from_store(traj_store(s, m.device), c.P, step).cpu().numpy()
        _check_update(m, c, hp, st, st0, batch, want, met, step, tgt0, tr, f"{case} update {u}:")
    print(f"{case}: {int(tr.excused.sum())} of {tr.excused.size} parameters excused from the element-wise check")   # shown by pytest -rP / -s
    m.close()


# ---- 5. determinism -----------------------------------------------------------------------------------------------------------------------------
def _state(m, c):
    vt, ret, adv = m.scratch(c.P, c.T)
    out = dict(theta=m.theta, theta_tgt=m.theta_tgt, adam_m=m.adam_m, adam_v=m.adam_v, grad=m.grad, metrics=m._metrics, vt=vt, ret=ret, adv=adv)
    out = {k: v.detach().cpu().clone() for k, v in out.items()}
    if m.standardise_returns:
        mean, var, count = m.ret_ms()
        out.update(ret_mean=mean, ret_var=var, ret_count=torch.tensor(count, dtype=torch.float64))
    return out


@pytest.mark.parametrize("case", ["ia2c_hard", "mappo_hard_standardise"])
def test_chain_is_deterministic(case):
    """two handles from the same initial state through the same chain end with the same bits in every state tensor; for A2C a third handle takes
    every update as marl_a2c_update_grads + marl_a2c_update_apply and ends bit-equal as well"""
    c = CHAIN[case]
    torch.manual_seed(11)
    ms = [_model(c) for _ in range(2 if c.ppo else 3)]
    _perturb_target(ms[0])
    for m in ms[1:]:
        m.theta.copy_(ms[0].theta); m.theta_tgt.copy_(ms[0].theta_tgt)
    for step, s in zip(c.steps, _chain_batches(c)):
        ts = traj_store(s, ms[0].device)
        ms[0].update_from_store(ts, c.P, step); ms[1].update_from_store(ts, c.P, step)
        if len(ms) > 2:
            ms[2].update_grads(ts, c.P); ms[2].update_apply(step)
    want = _state(ms[0], c)
    for i, m in enumerate(ms[1:], 1):
        got = _state(m, c)
        assert got.keys() == want.keys()
        for k in want:
            assert torch.equal(got[k], want[k]), f"handle {i}, {k}: max abs difference {float((got[k].double() - want[k].double()).abs().max()):.3e}"
    for m in ms:
        m.close()


# ---- 6. the training driver ----------------------------------------------------------------------------------------------------------------------
AC_COLS = ("environment_steps", "actor_loss", "entropy", "value_loss", "loss", "mean_episode_returns", "agent0/mean_episode_returns", "mean_episode_length", "updates")


@pytest.mark.parametrize("alg,flags", [("mappo", (True, True)), ("ia2c", (True, False)), ("ippo", (True, True))])
def test_driver_trains_recurrent_parts(tmp_path, monkeypatch, alg, flags):
    import pandas as pd

    from codebase_b200 import run

    monkeypatch.chdir(tmp_path)
    run.main([f"+algorithm={alg}", "env.name=lbforaging:Foraging-8x8-2p-3f-v3", "env.time_limit=25", "env.parallel_envs=256", "seed=1",
              f"algorithm.model.actor.use_rnn={flags[0]}", f"algorithm.model.critic.use_rnn={flags[1]}",
              "algorithm.total_steps=30000", "algorithm.eval_interval=6000", f"run_dir={tmp_path}/out"])
    df = pd.read_csv(tmp_path / "out" / "results.csv")
    for col in AC_COLS:
        assert col in df.columns, col
    assert len(df) >= 3 and df["environment_steps"].is_monotonic_increasing and np.isfinite(df["loss"]).all()
    assert df["mean_episode_length"].between(1, 25).all()


def test_collector_starts_every_collection_from_zero_h():
    """two collectors on two envs of the same seed record the same batch although one of them starts with hidden-state buffers left non-zero (as
    after an earlier collection): every collection starts the recurrent actor from h = 0 (ac/train.py:69-77)"""
    from codebase_b200.ac.train import Collector
    from codebase_b200.utils.envs import make_env

    c = Case(P=64, T=25)
    torch.manual_seed(2)
    m = _model(c)
    got = []
    for dirty in (False, True):
        env = make_env(5, name="lbforaging:Foraging-8x8-2p-3f-v3", time_limit=25, parallel_envs=64)
        col = Collector(env, m, 25)
        assert col.rnn
        if dirty:
            for h in col.h:
                h.copy_(torch.randn_like(h))
        col.collect()
        got.append({k: getattr(col.batch, k).cpu().clone() for k in ("obs", "act", "rew", "done", "filled")})
        env.close()
    for k in got[0]:
        assert torch.equal(got[0][k], got[1][k]), k
    assert int(got[0]["filled"].sum()) > 0
    m.close()


def test_checkpoint_eval_round_trip(tmp_path, monkeypatch):
    import os

    from codebase_b200 import eval as ev
    from codebase_b200 import run

    monkeypatch.chdir(tmp_path)
    out = f"{tmp_path}/out"
    run.main(["+algorithm=mappo", "env.name=lbforaging:Foraging-8x8-2p-3f-v3", "env.time_limit=25", "env.parallel_envs=256", "seed=0",
              "algorithm.model.actor.use_rnn=True", "algorithm.model.critic.use_rnn=True", "algorithm.total_steps=20000", "algorithm.eval_interval=6000",
              "algorithm.save_interval=6000", f"run_dir={out}"])
    monkeypatch.chdir(tmp_path)
    steps = sorted(int(f[7:-3]) for f in os.listdir(f"{out}/checkpoints"))
    sd = torch.load(f"{out}/checkpoints/model_s{steps[-1]}.pt", weights_only=True)
    assert tuple(sd["actor.independent.0.rnn.weight_hh_l0"].shape) == (384, 128)
    assert tuple(sd["critic.independent.1.first_layer.weight"].shape) == (128, 30) and "target_critic.independent.0.rnn.bias_ih_l0" in sd
    res = ev.main([f"path={out}", "episodes=32", "seed=3"])
    assert res["load_step"] == steps[-1] and res["episodes"] == 32 and np.isfinite(res["mean_episode_returns"])

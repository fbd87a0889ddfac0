"""GPU: the actor-critic learners (IA2C, MAA2C: marl_a2c_update; IPPO, MAPPO: marl_ppo_update) over K updates that are never re-synchronised
with the oracle.  The device state (parameters, Adam state and its step counter, target critic, running return statistics) evolves on its own;
the oracle (lr.a2c_update / lr.ppo_update) takes the same batches in step.  After every update the test checks the n-step returns, the target
critic's values, the advantages, the raw and clipped gradients, the metrics (losses, entropy, grad norm, filled count), Adam m / v per layer
block, the parameters element by element (except where Adam is ill-conditioned: an oracle gradient below 1e-4 of its block's largest on some
step so far; never an output-layer bias), the target critic's own update rule, and the running return statistics.

A second test runs two handles through the same chain and requires every state tensor to end equal bit for bit (fixed-order reductions)."""
import copy
import dataclasses

import numpy as np
import pytest
import torch

from oracle import learner_ref as lr
from tests.helpers import TIE, NearTie, ac_batch, ac_model, ac_oracle_batch, assert_grad_close, clipped, close_scaled, redraw_on_near_tie, traj_store

pytestmark = pytest.mark.gpu


@dataclasses.dataclass(frozen=True)
class Case:
    ppo: bool = False
    N: int = 2
    D: int = 15
    A: int = 6
    sharing: object = False
    centralised: bool = False
    P: int = 64                  # environments of each update (n_envs)
    cap: int = 0                 # store capacity and max_envs (0: P)
    T: int = 25
    steps: tuple = (0, 64, 128, 200)   # environment step of each update (hard syncs where step % tu == 0); K = len(steps)
    tu: float = 200              # target_update_interval_or_tau
    grad_clip: float = 0.0
    lr: float = 3e-4
    gamma: float = 0.99
    n_steps: int = 5
    vcoef: float = 0.5
    ecoef: float = 0.001
    epochs: int = 4
    standardise: bool = False
    rew_scale: float = 1.0
    clip_reached: bool = False   # PPO: the oracle's surrogate must block some entries' gradient in some epoch


# Each case covers something no other case does.
CASES = {
    # hard syncs hit (0, 200, 400) and missed (64, 128, 264); Adam's bias correction over 6 unglued steps
    "ia2c2_hard_syncs": Case(steps=(0, 64, 128, 200, 264, 400)),
    # 2 x value_loss_coef != 1, the entropy gradient at a visible weight, float32(gamma^k) away from 0.99, one-step returns
    "ia2c_coefs_nstep1": Case(vcoef=1.3, ecoef=0.05, gamma=0.9, n_steps=1),
    # n_steps == T: no bootstrap anywhere
    "ia2c_T7_nstep7": Case(T=7, n_steps=7, P=128),
    # n_steps = 64 = kMaxNStep > T: no bootstrap anywhere, the longest power table
    "ia2c_T7_nstep64": Case(T=7, n_steps=64, P=96),
    # n_steps = T - 1: the bootstrap reads the last observation only
    "ia2c_nstep24": Case(n_steps=24),
    # Polyak target; clipping active on every update (adam_kernel's own norm: 76 046 parameters, 2 mod 4, reach its scalar tail loop)
    "ia2c_polyak_clip_active": Case(tu=0.05, grad_clip=0.05),
    # full kOutPad head (A = 8); shared and independent networks in one set
    "ia2c3_shared010_A8": Case(N=3, sharing=(0, 1, 0), A=8, P=48),
    # a head narrower than 4 (A = 3); n_envs (40) below max_envs and the store's capacity (96)
    "ia2c_A3_P_below_max_envs": Case(A=3, P=40, cap=96),
    # the default IPPO path
    "ippo_default": Case(ppo=True, steps=(0, 3, 4), tu=2),
    # the clipped surrogate reached (small batch: few entries near the clip edges); Polyak once per update, clip_grad_norm_ active
    "ippo_clip_reached_polyak": Case(ppo=True, lr=3e-3, epochs=6, grad_clip=0.5, tu=0.05, P=16, T=10, steps=(0, 1, 2), clip_reached=True),
    # running return statistics carried unglued across PPO updates (returns away from the unit scale)
    "ippo_shared_standardise": Case(ppo=True, sharing=True, standardise=True, rew_scale=3.0, steps=(0, 3, 4), tu=2),
    # MAPPO: joint-row source modes 2 (training) / 3 inside a chain, with the running statistics
    "mappo_standardise": Case(ppo=True, centralised=True, standardise=True, steps=(0, 3, 4), tu=2, epochs=2),
    # MAA2C at the widest joint observation (2 x 16 = 32: KP = 32 tiles, tensor-core forward at 32)
    "maa2c_D16_joint32": Case(D=16, centralised=True),
}


def _hp(c):
    return lr.A2CHP(lr=c.lr, gamma=c.gamma, grad_clip=c.grad_clip, n_steps=c.n_steps, entropy_coef=c.ecoef, value_loss_coef=c.vcoef,
                    target_update_interval_or_tau=c.tu)


def _model(c):
    sharing = list(c.sharing) if isinstance(c.sharing, tuple) else c.sharing
    return ac_model(_hp(c), c.N, c.D, c.cap or c.P, c.T, A=c.A, sharing=sharing, cls="PPONetwork" if c.ppo else "A2CNetwork",
                    centralised=c.centralised, standardise=c.standardise, num_epochs=c.epochs)


def _perturb_target(m):
    """a target critic that differs from the critic until the first sync, so that the target's values and update rule matter"""
    m.theta_tgt.copy_(m.theta_tgt + 0.01 * torch.randn_like(m.theta_tgt))


def _batches(c):
    rng = np.random.default_rng(c.P * 7 + c.T * 3 + c.A + c.n_steps)
    for _ in c.steps:
        s = ac_batch(rng, c.cap or c.P, c.N, c.T, c.D, A=c.A)
        s["rew"] *= c.rew_scale
        yield s


def _blocks(m, c):
    """(name, slice) of every layer block of every actor and critic network in the flat [actor | critic] vector"""
    out = []
    o = 0
    for part, n_nets, ind, outd in (("actor", m.n_actor_nets, c.D, c.A), ("critic", m.n_critic_nets, m.critic_in, 1)):
        for k in range(n_nets):
            for name, size in zip(("W1", "b1", "W2", "b2", "W3", "b3"), (lr.H * ind, lr.H, lr.H * lr.H, lr.H, outd * lr.H, outd)):
                out.append((f"{part}{k}.{name}", slice(o, o + size)))
                o += size
    assert o == m.n_actor + m.n_critic
    return out


def _polyak_close(got, old, new, tau):
    """got == (1 - tau) old + tau new in float32, to 1 ulp of any of the three roundings (plain, or contracted to an FMA either way)"""
    t = np.float32(tau)
    a = np.float32(1) - t
    plain = (a * old + t * new).astype(np.float32)
    fma1 = (a.astype(np.float64) * old + (t * new).astype(np.float64)).astype(np.float32)
    fma2 = (t.astype(np.float64) * new + (a * old).astype(np.float64)).astype(np.float32)
    err = np.min([np.abs(got.astype(np.float64) - x) / np.spacing(np.abs(x)) for x in (plain, fma1, fma2)], axis=0)
    assert err.max() <= 1.0, f"Polyak target off by {err.max():.1f} ulp"


def _close(a, b, tol, what):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert np.allclose(a, b, rtol=tol, atol=tol), (what, float(np.abs(a - b).max()))


@pytest.mark.parametrize("case", list(CASES))
@redraw_on_near_tie
def test_chain_matches_oracle(case):
    c = CASES[case]
    hp = _hp(c)
    m = _model(c)
    _perturb_target(m)
    nets = list(m.actor_net)
    st = lr.A2CState(m.theta[: m.n_actor].cpu().clone(), m.theta[m.n_actor:].cpu().clone(), m.theta_tgt.cpu().clone(), nets, list(m.critic_net), c.D, c.A,
                     centralised=c.centralised, ret_ms=lr.RunningMeanStdRef((c.N,)) if c.standardise else None)
    n, na = m.n_actor + m.n_critic, m.n_actor
    blocks = _blocks(m, c)
    mtol = 2e-5 if c.ppo else 1e-5          # the metric bars of tests/test_ppo.py and tests/test_a2c_gpu.py
    gtol = 2e-5 if c.ppo or c.standardise else 1e-5
    ptol = 1e-5 * max(1.0, c.lr / 3e-4)     # the whole-vector 0.999-quantile bar of tests/test_ppo.py
    excused = np.zeros(n, bool)             # elements whose oracle gradient was ill-conditioned on some optimiser step so far
    abs_m = np.zeros(n)                     # Adam's m without cancellation: the same moving average of |clipped gradient|
    clip_seen = False
    for u, (step, s) in enumerate(zip(c.steps, _batches(c))):
        what = f"update {u}:"
        batch = ac_oracle_batch({k: v[: c.P] for k, v in s.items()})
        st0 = copy.deepcopy(st)
        if c.ppo:
            want = lr.ppo_update(st, batch, hp, step, c.epochs, 0.2)
            if min(want["clip_margin"]) < TIE:   # a ratio on the edge of the clip range: the surrogate's gradient jumps there
                raise NearTie(f"{what} a ratio {min(want['clip_margin']):.1e} from the edge of the clip range")
            clip_seen |= max(want["clip_frac"]) > 0
            raws = [np.concatenate([g["actor"].numpy(), g["critic"].numpy()]) for g in want["grads"]]
            steps_clipped = [np.concatenate([g["actor"].numpy(), g["critic"].numpy()]) for g in want["grads_clipped"]]
            want_clipped = np.concatenate([want["grads_clipped"][-1]["actor"].numpy(), want["grads_clipped"][-1]["critic"].numpy()])
            want_norm = float(np.mean(want["grad_norms"]))
            risk = lambda: lr.ppo_kink_risk(st0, batch, hp, want, 0.2)   # noqa: E731 -- the last epoch's loss, at the parameters it started from
        else:
            want = lr.a2c_update(st, batch, hp, step)
            raws = [np.concatenate([want["grad"]["actor"].numpy(), want["grad"]["critic"].numpy()])]
            want_clipped = np.concatenate([want["grad_clipped"]["actor"].numpy(), want["grad_clipped"]["critic"].numpy()])
            steps_clipped = [want_clipped]
            want_norm = want["grad_norm"]
            risk = lambda: lr.a2c_kink_risk(st0, batch, hp)   # noqa: E731
        tgt0 = m.theta_tgt.cpu().numpy().copy()
        met = m.update_from_store(traj_store(s, m.device), c.P, step).cpu().numpy()
        # n-step returns, target-critic values (before the statistics' rescaling), advantages
        vt, ret, adv = (x.cpu().numpy() for x in m.scratch(c.P, c.T))
        _close(ret, want["returns"].permute(2, 1, 0).numpy(), gtol, f"{what} returns")
        _close(vt, want["next_value"].permute(2, 1, 0).numpy(), 1e-5, f"{what} target values")
        if not c.ppo:
            _close(adv, want["advantages"].permute(2, 1, 0).numpy(), 1e-5, f"{what} advantages")
        # gradient of the (last) optimiser step, raw and clipped
        g = m.grad.cpu().numpy()
        fill = float(batch["filled"].sum())
        assert g[n + 1] == fill and met[4] == fill, (what, g[n + 1], met[4], fill)
        assert_grad_close(lr, st0, batch, hp, g[:n] / fill, raws[-1], tol=gtol, what=what, kink_risk=risk)
        close_scaled(clipped(g[:n] / fill, c.grad_clip), want_clipped, gtol)
        # metrics: losses and entropy (PPO: the epochs' means), the grad-norm metric, filled count (above)
        got = m.metrics_dict(torch.tensor(met))
        _close([got[k] for k in ("loss", "actor_loss", "value_loss", "entropy")], [want[k] for k in ("loss", "actor_loss", "value_loss", "entropy")], mtol, what)
        assert np.allclose(met[1], want_norm, rtol=1e-4, atol=1e-5), (what, met[1], want_norm)
        if c.grad_clip and c.grad_clip < 0.1:
            assert want_norm > c.grad_clip, "this case is meant to clip on every update"
        # Adam m / v, per layer block: every block is judged on its own scale, never on the whole vector's largest element.  v (a moving average
        # of g^2) is judged by close_scaled against its own largest |v|.  m is a signed moving average: where consecutive gradients change sign it
        # cancels, and its largest |m| stops measuring how precisely the device computed it (a one-element critic b3 cancelled to 1 % of its
        # gradient after one update, with the gradient itself agreeing to 2e-6).  So m's scale is the largest element of the same moving average
        # of |clipped g| in the block: equal to close_scaled's largest |m| where the gradients keep their sign, larger only where m cancels.
        for gc in steps_clipped:
            abs_m += (np.abs(gc) - abs_m) * (1 - 0.9)
        wm = np.concatenate([st.m["actor"].numpy(), st.m["critic"].numpy()]); wv = np.concatenate([st.v["actor"].numpy(), st.v["critic"].numpy()])
        am, av = m.adam_m.cpu().numpy(), m.adam_v.cpu().numpy()
        for name, sl in blocks:
            err = np.abs(am[sl].astype(np.float64) - wm[sl]).max()
            assert err <= gtol * abs_m[sl].max(), f"{what} Adam m of {name}: {err:.3e} > {gtol:g} x {abs_m[sl].max():.3e}"
            try:
                close_scaled(av[sl], wv[sl], 2 * gtol)
            except AssertionError as e:
                raise AssertionError(f"{what} Adam v of {name}: {e}") from None
        # parameters: the whole-vector quantile, then every element that Adam did not leave ill-conditioned
        for r in raws:
            for name, sl in blocks:
                low = np.abs(r[sl]) < 1e-4 * np.abs(r[sl]).max()
                if name.endswith("b3") and low.any():   # the oracle's own gradient, not the device's: an unlucky draw, re-drawn, never excused
                    raise NearTie(f"{what} the oracle's gradient of {name} is below 1e-4 of the block's largest: {np.abs(r[sl]).tolist()}")
                excused[sl] |= low
        th, want_th = m.theta.cpu().numpy(), np.concatenate([st.actor.numpy(), st.critic.numpy()])
        tg = m.theta_tgt.cpu().numpy()
        for name, mine, theirs, exc in (("theta", th, want_th, excused), ("target", tg, st.target.numpy(), excused[na:])):
            d = np.abs(mine - theirs)
            assert np.quantile(d, 0.999) < ptol and d.max() < 2 * c.lr * (c.epochs if c.ppo else 1) * (u + 1) + 1e-6, (what, name, np.quantile(d, 0.999), d.max())
            bad = np.flatnonzero((d > 1e-5) & ~exc)
            assert bad.size == 0, f"{what} {name}: {bad.size} elements off by up to {d[bad].max():.2e} (first {bad[:5]})"
        # the target critic, on the device alone
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
    print(f"{case}: {int(excused.sum())} of {n} parameters excused from the element-wise check")   # shown by pytest -rP / -s
    if c.clip_reached:
        assert clip_seen, "the clipped surrogate was never reached"
    m.close()


def _state(m, c):
    vt, ret, adv = m.scratch(c.P, c.T)
    out = dict(theta=m.theta, theta_tgt=m.theta_tgt, adam_m=m.adam_m, adam_v=m.adam_v, grad=m.grad, metrics=m._metrics, vt=vt, ret=ret, adv=adv)
    out = {k: v.detach().cpu().clone() for k, v in out.items()}
    if m.standardise_returns:
        mean, var, count = m.ret_ms()
        out.update(ret_mean=mean, ret_var=var, ret_count=torch.tensor(count, dtype=torch.float64))
    return out


@pytest.mark.parametrize("case", ["ia2c2_hard_syncs", "ippo_shared_standardise"])
def test_chain_is_deterministic(case):
    """two handles from the same initial state through the same chain end with the same bits in every state tensor"""
    c = CASES[case]
    torch.manual_seed(11)
    a = _model(c)
    _perturb_target(a)
    b = _model(c)
    b.theta.copy_(a.theta); b.theta_tgt.copy_(a.theta_tgt)
    for step, s in zip(c.steps, _batches(c)):
        for m in (a, b):
            m.update_from_store(traj_store(s, m.device), c.P, step)
    got, want = _state(a, c), _state(b, c)
    assert got.keys() == want.keys()
    for k in want:
        assert torch.equal(got[k], want[k]), f"{k}: max abs difference {float((got[k].double() - want[k].double()).abs().max()):.3e}"
    a.close(); b.close()

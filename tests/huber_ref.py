"""The Huber TD loss of IDQN, VDN and QMIX (algorithm.huber_delta) restated for the tests, in float64.  TEST INFRASTRUCTURE ONLY.

The reference's losses are torch.nn.functional.mse_loss(chosen, returns, reduction="none") of the TD error d = Q - y, summed over agents for IDQN,
then the filled-masked mean (marlbase/dqn/model.py:160-163, 266-269, 424-427).  With algorithm.huber_delta = δ the project replaces mse_loss by
torch.nn.functional.huber_loss(..., delta=δ) (DESIGN.md §4.4e), i.e. per element

    0.5 d²  if |d| < δ,   else  δ (|d| - 0.5 δ),

which `huber` states from that definition (no torch loss function).  `dqn_td` / `qmix_td` are oracle.learner_ref.dqn_loss and
tests/qmix_options_ref.qmix_loss up to the TD error, with the returns of tests/td_lambda_ref.py (`lam` None: the one-step target), in float64 (the
running statistics of standardise_returns stay the reference's float32 RunningMeanStd, which absorbs float32 returns); `dqn_loss` / `qmix_loss` apply
`huber` to them, and `huber_in(delta, lam)` runs learner_ref's / qmix_ref's updates and ReLU-kink bounds with those losses.
"""
from __future__ import annotations

import contextlib
import copy
import dataclasses
import functools

import torch

from oracle import learner_ref as lr
from oracle import qmix_ref as qr
from tests import qmix_options_ref as qo
from tests import td_lambda_ref as tl


def huber(d, delta):
    """per-element Huber loss of the TD errors d with threshold delta (float64 when d is)"""
    a = d.abs()
    return torch.where(a < delta, 0.5 * d * d, delta * (a - 0.5 * delta))


def _standardise(returns, ret_ms):
    ret_ms.update(returns.float())
    return (returns - ret_ms.mean.to(returns.dtype)) / torch.sqrt(ret_ms.var.to(returns.dtype))


def dqn_td(theta, theta_tgt, agent_net, in_dim, out_dim, batch, hp: lr.DqnHP, ret_ms=None, lam=None):
    """the TD errors Q - y of learner_ref.dqn_loss in float64: IDQN (N, T, B), one column per agent; VDN (T, B), all agents with agent 0's reward"""
    th = theta.double()
    obss = batch["obss"].double()
    rewards, dones, filled = (batch[k].double() for k in ("rewards", "dones", "filled"))
    lam = 0.0 if lam is None else lam
    q = torch.stack(lr.agents_forward(th, agent_net, list(obss), in_dim, out_dim))          # (N,T+1,B,A)
    chosen = q[:, :-1].gather(-1, batch["actions"].unsqueeze(-1)).squeeze(-1)                 # (N,T,B)
    with torch.no_grad():
        tq = torch.stack(lr.agents_forward(theta_tgt.double(), agent_net, list(obss), in_dim, out_dim))[:, 1:]
        if hp.double_q:
            target = tq.gather(-1, q.detach()[:, 1:].argmax(-1, keepdim=True)).squeeze(-1)
        else:
            target = tq.max(-1)[0]
    if hp.mixer == 1:
        chosen, target = chosen.sum(0), target.sum(0)
        if ret_ms is not None:
            target = target * torch.sqrt(ret_ms.var.double()) + ret_ms.mean.double()
        returns = tl.lambda_targets(rewards[0], dones, filled, target, lam, hp.gamma)       # (T,B)
        if ret_ms is not None:
            returns = _standardise(returns, ret_ms)
        return chosen - returns.detach()
    if ret_ms is not None:
        target = (target.permute(1, 2, 0) * torch.sqrt(ret_ms.var.double()) + ret_ms.mean.double()).permute(2, 0, 1)
    returns = tl.lambda_targets(rewards.permute(1, 0, 2), dones, filled, target.permute(1, 0, 2), lam, hp.gamma).permute(1, 0, 2)   # (N,T,B)
    if ret_ms is not None:
        returns = _standardise(returns.permute(1, 2, 0), ret_ms).permute(2, 0, 1)
    return chosen - returns.detach()


def qmix_td(theta, mix, st: qo.QmixOptState, batch, hp: lr.DqnHP, lam=None):
    """the TD errors Q_tot - y (T, B) of tests/qmix_options_ref.qmix_loss (either mixer, standardise_returns) in float64"""
    obss = batch["obss"].double()
    rewards, dones, filled = (batch[k].double() for k in ("rewards", "dones", "filled"))
    N, hl = obss.shape[0], st.hypernet_layers
    q = torch.stack(lr.agents_forward(theta.double(), st.agent_net, list(obss), st.in_dim, st.out_dim))
    chosen = q[:, :-1].gather(-1, batch["actions"].unsqueeze(-1)).squeeze(-1)
    chosen = qo.mixer_forward(mix.double(), chosen, torch.concat(list(obss[:, :-1]), dim=-1), N, st.embed_dim, st.hypernet_embed, hl)
    with torch.no_grad():
        tq = torch.stack(lr.agents_forward(st.theta_tgt.double(), st.agent_net, list(obss), st.in_dim, st.out_dim))[:, 1:]
        if hp.double_q:
            target = tq.gather(-1, q.detach()[:, 1:].argmax(-1, keepdim=True)).squeeze(-1)
        else:
            target = tq.max(-1)[0]
        target = qo.mixer_forward(st.mix_tgt.double(), target, torch.concat(list(obss[:, 1:]), dim=-1), N, st.embed_dim, st.hypernet_embed, hl)
    if st.ret_ms is not None:
        target = target * torch.sqrt(st.ret_ms.var.double()) + st.ret_ms.mean.double()
    returns = tl.lambda_targets(rewards[0], dones, filled, target, 0.0 if lam is None else lam, hp.gamma)
    if st.ret_ms is not None:
        returns = _standardise(returns, st.ret_ms)
    return chosen - returns.detach()


def _mean(loss, filled):
    return (loss * filled).sum() / filled.sum()


def dqn_loss(theta, theta_tgt, agent_net, in_dim, out_dim, batch, hp: lr.DqnHP, ret_ms=None, delta=1.0, lam=None):
    """learner_ref.dqn_loss with the Huber TD loss (IDQN: summed over agents, then the filled-masked mean), float64"""
    loss = huber(dqn_td(theta, theta_tgt, agent_net, in_dim, out_dim, batch, hp, ret_ms, lam), delta)
    return _mean(loss if hp.mixer == 1 else loss.sum(0), batch["filled"].double())


def qmix_loss(theta, mix, st: qo.QmixOptState, batch, hp: lr.DqnHP, delta=1.0, lam=None):
    """tests/qmix_options_ref.qmix_loss with the Huber TD loss of Q_tot, float64"""
    return _mean(huber(qmix_td(theta, mix, st, batch, hp, lam), delta), batch["filled"].double())


@contextlib.contextmanager
def huber_in(delta, lam=None):
    """learner_ref.dqn_update / dqn_kink_risk and qmix_ref.qmix_update with the Huber losses of `delta` (None: unchanged, the squared error) and
    the TD(λ) target of `lam` (None: the one-step target)"""
    if delta is None:
        with tl.td_lambda_in(lam):
            yield
        return
    saved = lr.dqn_loss, qr.qmix_loss
    lr.dqn_loss = functools.partial(dqn_loss, delta=delta, lam=lam)
    qr.qmix_loss = functools.partial(qmix_loss, delta=delta, lam=lam)
    try:
        yield
    finally:
        lr.dqn_loss, qr.qmix_loss = saved


def qmix_kink_risk(st: qo.QmixOptState, batch, hp: lr.DqnHP, delta, lam=None):
    """qmix_options_ref.qmix_kink_risk of the Huber loss"""
    return lr.kink_risk(lambda th: qmix_loss(th, st.mix, dataclasses.replace(st, ret_ms=copy.deepcopy(st.ret_ms)), batch, hp, delta, lam), st.theta)


def branches(d, filled, delta):
    """(filled TD errors inside the band |d| < delta, filled TD errors outside it): d (..., T, B), filled (T, B)"""
    m = filled.double().expand_as(d) > 0
    inside = (d.detach().abs() < delta) & m
    return int(inside.sum()), int(m.sum()) - int(inside.sum())


# ---- the golden cases (tests/golden/huber_reference.npz, written by tests/golden/make_huber_golden.py from the reference's own learners) ----------
@dataclasses.dataclass(frozen=True)
class GoldenCase:
    cls: str                    # the reference's learner class
    delta: float
    hl: int = 2                 # QMIX: mixing.hypernet_layers
    sharing: bool = False
    double_q: bool = True
    N: int = 2
    D: int = 9
    seed: int = 0


GOLDEN_A, GOLDEN_T, GOLDEN_B, GOLDEN_UPDATES = 6, 6, 16, 3
GOLDEN_CASES = {
    "idqn_indep": GoldenCase("QNetwork", 0.5, seed=41),
    "idqn_shared_single_q": GoldenCase("QNetwork", 1.0, sharing=True, double_q=False, N=3, seed=42),
    "vdn": GoldenCase("VDNetwork", 1.0, seed=43),
    "qmix_h1": GoldenCase("QMixNetwork", 12.0, hl=1, N=3, seed=44),
    "qmix_h2": GoldenCase("QMixNetwork", 1.0, seed=45),
}


def golden_hp(c: GoldenCase):
    return lr.DqnHP(double_q=c.double_q, target_update_interval_or_tau=2, mixer=1 if c.cls == "VDNetwork" else 0)


def golden_state(c: GoldenCase):
    """the case's initial networks: the oracle and the reference (fixture generation) start from these"""
    n_nets = 1 if c.sharing else c.N
    theta = lr.init_flat(n_nets, c.D, GOLDEN_A, generator=torch.Generator().manual_seed(c.seed))
    agent_net = [0] * c.N if c.sharing else list(range(c.N))
    if c.cls != "QMixNetwork":
        return lr.DqnState(theta.clone(), theta.clone(), agent_net, c.D, GOLDEN_A)
    torch.manual_seed(c.seed)
    mix = qo.init_mixer_flat(c.N, c.N * c.D, 64, 32, c.hl)
    return qo.QmixOptState(theta.clone(), theta.clone(), mix.clone(), mix.clone(), agent_net, c.D, GOLDEN_A, hypernet_layers=c.hl)


def golden_batches(c: GoldenCase):
    """GOLDEN_UPDATES batches (N, T+1, B, D): dense rewards of spread 1.5 (team rewards for VDN and QMIX) so that TD errors fall on both sides of
    delta, a few terminal steps and unfilled rows"""
    g = torch.Generator().manual_seed(1000 + c.seed)
    N, T, B = c.N, GOLDEN_T, GOLDEN_B
    out = []
    for _ in range(GOLDEN_UPDATES):
        rew = 1.5 * torch.randn(N, T, B, generator=g)
        if c.cls != "QNetwork":
            rew[:] = rew[:1]
        out.append(dict(obss=torch.randn(N, T + 1, B, c.D, generator=g), actions=torch.randint(0, GOLDEN_A, (N, T, B), generator=g), rewards=rew,
                        dones=(torch.rand(T + 1, B, generator=g) < 0.05).float(), filled=(torch.rand(T, B, generator=g) < 0.9).float()))
    return out


def golden_update(c: GoldenCase, st, batch, hp, delta=None):
    """one oracle update of a golden case with the Huber loss of `delta` (default: the case's)"""
    with huber_in(c.delta if delta is None else delta):
        return qr.qmix_update(st, batch, hp) if c.cls == "QMixNetwork" else lr.dqn_update(st, batch, hp)


def golden_td(c: GoldenCase, st, batch, hp):
    """the TD errors of the case's next update (for the branch counts)"""
    if c.cls == "QMixNetwork":
        return qmix_td(st.theta, st.mix, st, batch, hp)
    return dqn_td(st.theta, st.theta_tgt, st.agent_net, st.in_dim, st.out_dim, batch, hp)

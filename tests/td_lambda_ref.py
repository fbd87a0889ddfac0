"""TD(λ) targets of IDQN, VDN and QMIX (algorithm.td_lambda) restated for the tests, in float64.  TEST INFRASTRUCTURE ONLY.

The reference has only the one-step target r_t + γ (1 - d_{t+1}) v_{t+1}; the project defines the TD(λ) target (DESIGN.md §4.4d) per column (IDQN:
an agent; VDN and QMIX: the team) of a sampled episode, with f_T := 0, as

    G_t = r_t + γ (1 - d_{t+1}) ((1 - λ f_{t+1}) v_{t+1} + λ f_{t+1} G_{t+1})

i.e. the mixture (1 - λ) Σ_{n<L} λ^(n-1) G_t^(n) + λ^(L-1) G_t^(L) of the n-step returns, truncated at the first unfilled row t + L after t.
`lambda_targets` is the recursion (torch, any dtype); `lambda_mixture` evaluates the mixture from the definition of each G^(n) (numpy float64,
O(T²) per sequence) and shares no arithmetic with it.

`dqn_loss` / `qmix_loss` are oracle.learner_ref.dqn_loss and tests/qmix_options_ref.qmix_loss with G in place of the one-step returns, evaluated in
float64 (the running statistics of standardise_returns stay the reference's float32 RunningMeanStd); `td_lambda_in(lam)` runs learner_ref's /
qmix_ref's updates and ReLU-kink bounds with them.  At λ = 0 they are the reference's losses (tests/test_td_lambda.py), which the goldens pin.
"""
from __future__ import annotations

import contextlib
import copy
import dataclasses
import functools

import numpy as np
import torch

from oracle import learner_ref as lr
from oracle import qmix_ref as qr
from tests import qmix_options_ref as qo


def lambda_targets(rewards, dones, filled, boot, lam, gamma):
    """G (T, ...) by the backward recursion: rewards, filled, boot (T, ...) with boot[t] = v_{t+1}; dones (T+1, ...); trailing dimensions
    broadcast.  In boot's dtype."""
    T = boot.shape[0]
    r, d, f = (x.to(boot.dtype) for x in (rewards, dones, filled))
    out, nxt = [None] * T, torch.zeros_like(boot[0])
    for t in reversed(range(T)):
        live, f1 = 1.0 - d[t + 1], f[t + 1] if t + 1 < T else torch.zeros_like(f[0])
        nxt = r[t] + gamma * live * ((1.0 - lam * f1) * boot[t] + lam * f1 * nxt)
        out[t] = nxt
    return torch.stack(out)


def lambda_mixture(rewards, dones, filled, boot, lam, gamma):
    """the same G from the n-step returns G_t^(n) = Σ_{k<n} γ^k c_k r_{t+k} + γ^n c_n v_{t+n}, c_k = Π_{j=1..k} (1 - d_{t+j}), float64 numpy;
    all arrays share their trailing shape"""
    r, v = np.asarray(rewards, np.float64), np.asarray(boot, np.float64)
    T = r.shape[0]
    d, f = np.asarray(dones, np.float64).reshape(T + 1, -1), np.asarray(filled, np.float64).reshape(T, -1)
    r, v = r.reshape(T, -1), v.reshape(T, -1)
    out = np.zeros_like(r)
    for m in range(r.shape[1]):
        for t in range(T):
            L = 1
            while t + L < T and f[t + L, m] > 0:
                L += 1
            acc, c, g = 0.0, 1.0, 0.0
            for n in range(1, L + 1):
                acc += gamma ** (n - 1) * c * r[t + n - 1, m]
                c *= 1.0 - d[t + n, m]
                Gn = acc + gamma ** n * c * v[t + n - 1, m]
                g += (lam ** (L - 1) if n == L else (1.0 - lam) * lam ** (n - 1)) * Gn
            out[t, m] = g
    return out.reshape(np.asarray(rewards).shape)


def _standardised(returns, ret_ms):
    """RunningMeanStd step on the float32 returns (the device's statistics see float32 returns), then the returns standardised in float64"""
    ret_ms.update(returns.float())
    return (returns - ret_ms.mean.to(returns.dtype)) / torch.sqrt(ret_ms.var.to(returns.dtype))


def dqn_loss(theta, theta_tgt, agent_net, in_dim, out_dim, batch, hp: lr.DqnHP, ret_ms=None, lam=0.0):
    """learner_ref.dqn_loss with the TD(λ) target, in float64: IDQN one column per agent, VDN one column of all agents with agent 0's reward"""
    th = theta.double()
    obss = batch["obss"].double()
    rewards, dones, filled = (batch[k].double() for k in ("rewards", "dones", "filled"))
    N = obss.shape[0]
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
        returns = lambda_targets(rewards[0], dones, filled, target, lam, hp.gamma)           # (T,B)
        if ret_ms is not None:
            returns = _standardised(returns, ret_ms)
        loss = (chosen - returns.detach()) ** 2
    else:
        if ret_ms is not None:
            target = (target.permute(1, 2, 0) * torch.sqrt(ret_ms.var.double()) + ret_ms.mean.double()).permute(2, 0, 1)
        returns = lambda_targets(rewards.permute(1, 0, 2), dones, filled, target.permute(1, 0, 2), lam, hp.gamma).permute(1, 0, 2)   # (N,T,B)
        if ret_ms is not None:
            returns = _standardised(returns.permute(1, 2, 0), ret_ms).permute(2, 0, 1)
        loss = ((chosen - returns.detach()) ** 2).sum(0)
    return (loss * filled).sum() / filled.sum()


def qmix_loss(theta, mix, st: qo.QmixOptState, batch, hp: lr.DqnHP, lam=0.0):
    """tests/qmix_options_ref.qmix_loss (either mixer, standardise_returns) with the TD(λ) target of Q_tot, in float64"""
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
    returns = lambda_targets(rewards[0], dones, filled, target, lam, hp.gamma)
    if st.ret_ms is not None:
        returns = _standardised(returns, st.ret_ms)
    loss = (chosen - returns.detach()) ** 2
    return (loss * filled).sum() / filled.sum()


@contextlib.contextmanager
def td_lambda_in(lam):
    """learner_ref.dqn_update / dqn_kink_risk and qmix_ref.qmix_update with the TD(λ) losses of `lam` (None: unchanged, the one-step target)"""
    if lam is None:
        yield
        return
    saved = lr.dqn_loss, qr.qmix_loss
    lr.dqn_loss, qr.qmix_loss = functools.partial(dqn_loss, lam=lam), functools.partial(qmix_loss, lam=lam)
    try:
        yield
    finally:
        lr.dqn_loss, qr.qmix_loss = saved


def qmix_kink_risk(st: qo.QmixOptState, batch, hp: lr.DqnHP, lam):
    """qmix_options_ref.qmix_kink_risk of the TD(λ) loss"""
    return lr.kink_risk(lambda th: qmix_loss(th, st.mix, dataclasses.replace(st, ret_ms=copy.deepcopy(st.ret_ms)), batch, hp, lam), st.theta)

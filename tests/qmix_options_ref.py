"""CPU restatement of QMIX's two remaining reference options on top of oracle/qmix_ref.py.  TEST INFRASTRUCTURE ONLY.

Restated from (path:line in the reference project's marlbase/):
  dqn/model.py:283-285   QMixer with hypernet_layers == 1: hyper_w_1 = Linear(S, N*E), hyper_w_final = Linear(S, E) (hypernet_embed unused)
  dqn/model.py:357-358   standardise_returns: ret_ms = RunningMeanStd(shape=(1,)), one statistic per batch column once it has seen (T, B) returns
  dqn/model.py:415-422   target de-standardised with the statistics so far, the returns update them, the standardised returns enter the loss

The one-layer mixer's flat parameters follow the reference's state_dict order: hyper_w_1.{weight [N*E,S], bias}, hyper_w_final.{weight [E,S], bias},
hyper_b_1, V.0, V.2.  The two-layer form is oracle/qmix_ref.py's own.  The update, Adam, the target updates and the ReLU-kink bound are
qmix_ref's / learner_ref's functions run with this module's loss in place of qmix_ref.qmix_loss (`options()`), so both mixers share every line of
that arithmetic; recurrent agent networks combine with it through oracle.gru_ref.recurrent().  Pinned against outputs of the reference's
QMixNetwork by tests/test_qmix_options.py (tests/golden/qmix_options_reference.npz).
"""
from __future__ import annotations

import contextlib
import copy
import dataclasses
from dataclasses import dataclass

import torch
import torch.nn.functional as F

from oracle import learner_ref as lr
from oracle import qmix_ref as qr

MIXER_KEYS_1 = ("hyper_w_1", "hyper_w_final", "hyper_b_1", "V.0", "V.2")


def mixer_keys(hypernet_layers=2):
    if hypernet_layers not in (1, 2):   # the reference's QMixer raises for any other value (dqn/model.py:298-301)
        raise ValueError(f"hypernet_layers={hypernet_layers}: QMixer has 1 or 2 hypernetwork layers")
    return qr.MIXER_KEYS if hypernet_layers == 2 else MIXER_KEYS_1


def mixer_shapes(n_agents, state_dim, embed_dim, hypernet_embed, hypernet_layers=2):
    mixer_keys(hypernet_layers)
    if hypernet_layers == 2:
        return qr.mixer_shapes(n_agents, state_dim, embed_dim, hypernet_embed)
    N, S, E = n_agents, state_dim, embed_dim
    return ((N * E, S), (E, S), (E, S), (E, S), (1, E))


def mixer_size(n_agents, state_dim, embed_dim, hypernet_embed, hypernet_layers=2):
    return sum(o * i + o for o, i in mixer_shapes(n_agents, state_dim, embed_dim, hypernet_embed, hypernet_layers))


def split_mixer(flat, n_agents, state_dim, embed_dim, hypernet_embed, hypernet_layers=2):
    out, o = [], 0
    for (no, ni) in mixer_shapes(n_agents, state_dim, embed_dim, hypernet_embed, hypernet_layers):
        out.append(flat[o:o + no * ni].view(no, ni)); o += no * ni
        out.append(flat[o:o + no]); o += no
    return out


def mixer_flat_from_state_dict(sd, prefix="mixer", hypernet_layers=2):
    return torch.cat([sd[f"{prefix}.{k}.{p}"].reshape(-1) for k in mixer_keys(hypernet_layers) for p in ("weight", "bias")]).clone().float()


def mixer_state_dict_from_flat(flat, prefix, n_agents, state_dim, embed_dim, hypernet_embed, hypernet_layers=2):
    parts = split_mixer(flat, n_agents, state_dim, embed_dim, hypernet_embed, hypernet_layers)
    sd = {}
    for j, k in enumerate(mixer_keys(hypernet_layers)):
        sd[f"{prefix}.{k}.weight"] = parts[2 * j].clone(); sd[f"{prefix}.{k}.bias"] = parts[2 * j + 1].clone()
    return sd


def init_mixer_flat(n_agents, state_dim, embed_dim, hypernet_embed, hypernet_layers=2):
    """QMixer builds plain nn.Linear layers (PyTorch's default initialisation), in state_dict order."""
    parts = []
    for (no, ni) in mixer_shapes(n_agents, state_dim, embed_dim, hypernet_embed, hypernet_layers):
        lin = torch.nn.Linear(ni, no)
        parts += [lin.weight.data.reshape(-1), lin.bias.data.reshape(-1)]
    return torch.cat(parts).float()


def mixer_forward(flat, agent_qs, states, n_agents, embed_dim, hypernet_embed, hypernet_layers=2):
    """agent_qs (N, T, B), states (T, B, S) -> Q_tot (T, B)   (dqn/model.py:314-340)"""
    if hypernet_layers == 2:
        return qr.mixer_forward(flat, agent_qs, states, n_agents, embed_dim, hypernet_embed)
    N, T, B = agent_qs.shape
    S = states.shape[-1]
    w1w, b1w, wfw, bfw, wb, bb, wva, bva, wvb, bvb = split_mixer(flat, n_agents, S, embed_dim, hypernet_embed, 1)
    qs = agent_qs.permute(1, 2, 0).reshape(T * B, 1, N)
    x = states.reshape(-1, S)
    w1 = torch.abs(F.linear(x, w1w, b1w)).view(-1, N, embed_dim)
    b1 = F.linear(x, wb, bb).view(-1, 1, embed_dim)
    hidden = F.elu(torch.bmm(qs, w1) + b1)
    wf = torch.abs(F.linear(x, wfw, bfw)).view(-1, embed_dim, 1)
    v = F.linear(F.relu(F.linear(x, wva, bva)), wvb, bvb).view(-1, 1, 1)
    return (torch.bmm(hidden, wf) + v).view(T, B)


@dataclass
class QmixOptState(qr.QmixState):
    hypernet_layers: int = 2
    ret_ms: object = None      # learner_ref.RunningMeanStdRef((1,)) when cfg.standardise_returns (dqn/model.py:357-358), else None


def qmix_loss(theta, mix, st: QmixOptState, batch, hp: lr.DqnHP):
    """qmix_ref.qmix_loss with either mixer and the reference's return standardisation"""
    obss, actions, rewards, dones, filled = (batch[k] for k in ("obss", "actions", "rewards", "dones", "filled"))
    N, hl = obss.shape[0], st.hypernet_layers
    q = torch.stack(lr.agents_forward(theta, st.agent_net, list(obss), st.in_dim, st.out_dim))            # (N, T+1, B, A)
    chosen = q[:, :-1].gather(-1, actions.unsqueeze(-1)).squeeze(-1)
    chosen = mixer_forward(mix, chosen, torch.concat(list(obss[:, :-1]), dim=-1), N, st.embed_dim, st.hypernet_embed, hl)
    with torch.no_grad():
        tq = torch.stack(lr.agents_forward(st.theta_tgt, st.agent_net, list(obss), st.in_dim, st.out_dim))[:, 1:]
        if hp.double_q:
            target = tq.gather(-1, q.detach()[:, 1:].argmax(-1, keepdim=True)).squeeze(-1)
        else:
            target = tq.max(-1)[0]
        target = mixer_forward(st.mix_tgt, target, torch.concat(list(obss[:, 1:]), dim=-1), N, st.embed_dim, st.hypernet_embed, hl)
    if st.ret_ms is not None:                                            # dqn/model.py:415-416
        target = target * torch.sqrt(st.ret_ms.var) + st.ret_ms.mean
    returns = rewards[0] + hp.gamma * target * (1 - dones[1:])
    if st.ret_ms is not None:                                            # dqn/model.py:420-422: update() reshapes the (T, B) returns with reshape(-1, B)
        st.ret_ms.update(returns)
        returns = (returns - st.ret_ms.mean) / torch.sqrt(st.ret_ms.var)
    loss = (chosen - returns.detach()) ** 2
    return (loss * filled).sum() / filled.sum()


@contextlib.contextmanager
def options():
    """run qmix_ref.qmix_update with this module's loss"""
    saved = qr.qmix_loss
    qr.qmix_loss = qmix_loss
    try:
        yield
    finally:
        qr.qmix_loss = saved


def qmix_update(st: QmixOptState, batch, hp: lr.DqnHP):
    with options():
        return qr.qmix_update(st, batch, hp)


def qmix_kink_risk(st: QmixOptState, batch, hp: lr.DqnHP):
    """learner_ref.kink_risk of the agents' networks through the mixer; the loss reads (and advances) the running statistics, so every
    evaluation gets a copy of them"""
    return lr.kink_risk(lambda th: qmix_loss(th, st.mix, dataclasses.replace(st, ret_ms=copy.deepcopy(st.ret_ms)), batch, hp), st.theta)

"""CPU restatement (PyTorch float32, autograd) of the recurrent agent networks of the DQN family.  TEST INFRASTRUCTURE ONLY.

Restated from (path:line in the reference project's marlbase/):
  utils/models.py:51-116     RNNNetwork: first_layer Linear + ReLU, nn.GRU (one layer, sequence-first), final_layer Linear
  utils/models.py:119-130    make_network (dims = [D, 128, 128, A] -> one GRU layer)
  dqn/model.py:94-116        act carries the hiddens;  :127,133 training passes start from hiddens=None (zeros)

Over FLAT parameter vectors in the device layout ([n_nets][P], reference state_dict order).  The losses, the update, the double-Q margin and the
ReLU-kink bound are learner_ref's and qmix_ref's own functions run with this module's agents_forward in place of the MLP's (`recurrent()`), so
the recurrent learners share every line of loss arithmetic with the feed-forward ones.
"""
from __future__ import annotations

import contextlib
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import learner_ref as lr
from oracle import qmix_ref as qr

H = 128
NAMES = ("first_layer.weight", "first_layer.bias", "rnn.weight_ih_l0", "rnn.weight_hh_l0", "rnn.bias_ih_l0", "rnn.bias_hh_l0",
         "final_layer.weight", "final_layer.bias")


def shapes(in_dim, out_dim):
    return ((H, in_dim), (H,), (3 * H, H), (3 * H, H), (3 * H,), (3 * H,), (out_dim, H), (out_dim,))


def net_size(in_dim, out_dim):
    return sum(int(np.prod(s)) for s in shapes(in_dim, out_dim))


def split_net(flat, in_dim, out_dim):
    out, o = [], 0
    for shape in shapes(in_dim, out_dim):
        n = int(np.prod(shape))
        out.append(flat[o:o + n].view(*shape))
        o += n
    return out


def flat_from_state_dict(sd, prefix, n_nets):
    return torch.cat([sd[f"{prefix}.{k}.{name}"].reshape(-1) for k in range(n_nets) for name in NAMES]).clone().float()


def state_dict_from_flat(flat, prefix, n_nets, in_dim, out_dim):
    P, sd = net_size(in_dim, out_dim), {}
    for k in range(n_nets):
        for name, t in zip(NAMES, split_net(flat[k * P:(k + 1) * P], in_dim, out_dim)):
            sd[f"{prefix}.{k}.{name}"] = t.clone()
    return sd


def init_flat(n_nets, in_dim, out_dim, orthogonal=True):
    """RNNNetwork.__init__: first_layer and the GRU keep PyTorch's defaults, use_orthogonal_init touches final_layer only (global RNG)."""
    parts = []
    for _ in range(n_nets):
        first, gru, final = torch.nn.Linear(in_dim, H), torch.nn.GRU(H, H, num_layers=1), torch.nn.Linear(H, out_dim)
        if orthogonal:
            torch.nn.init.orthogonal_(final.weight.data, gain=math.sqrt(2))
            torch.nn.init.constant_(final.bias.data, 0)
        parts += [t.data.reshape(-1) for t in (first.weight, first.bias, gru.weight_ih_l0, gru.weight_hh_l0, gru.bias_ih_l0, gru.bias_hh_l0,
                                              final.weight, final.bias)]
    return torch.cat(parts).float()


def gru_net(flat_net, x, in_dim, out_dim, h0=None):
    """x (L, B, in_dim) -> q (L, B, out_dim), h (L, B, 128): every step's hidden state; h0 (B, 128) or None = zeros."""
    w1, b1, wih, whh, bih, bhh, w3, b3 = split_net(flat_net, in_dim, out_dim)
    z1 = F.linear(x, w1, b1)
    x1 = F.relu(z1)
    if lr._TAPS is not None and flat_net.requires_grad:   # learner_ref.kink_risk: the first layer's ReLU is the net's only kink
        x1.retain_grad()
        lr._TAPS.append((z1, x1, x))
    gi = F.linear(x1, wih, bih)
    h = torch.zeros(x.shape[1], H, dtype=x.dtype) if h0 is None else h0
    hs = []
    for t in range(x.shape[0]):
        gh = F.linear(h, whh, bhh)
        r = torch.sigmoid(gi[t, :, :H] + gh[:, :H])
        z = torch.sigmoid(gi[t, :, H:2 * H] + gh[:, H:2 * H])
        n = torch.tanh(gi[t, :, 2 * H:] + r * gh[:, 2 * H:])
        h = (1 - z) * n + z * h
        hs.append(h)
    hs = torch.stack(hs)
    return F.linear(hs, w3, b3), hs


def agents_forward(flat, agent_net, xs, in_dim, out_dim):
    """learner_ref.agents_forward for recurrent networks: xs per agent (T+1, B, D), each sequence from the zero state."""
    P = net_size(in_dim, out_dim)
    return [gru_net(flat[k * P:(k + 1) * P], x, in_dim, out_dim)[0] for k, x in zip(agent_net, xs)]


def act_steps(flat, agent_net, obs, in_dim, out_dim, h0=None):
    """model.act over consecutive steps: obs (S, E, N, D), h0 (E, N, 128) or None -> q (S, E, N, A), h (S, E, N, 128) after every step."""
    P = net_size(in_dim, out_dim)
    qs, hs = [], []
    for a, k in enumerate(agent_net):
        q, h = gru_net(flat[k * P:(k + 1) * P], obs[:, :, a], in_dim, out_dim, None if h0 is None else h0[:, a])
        qs.append(q); hs.append(h)
    return torch.stack(qs, 2), torch.stack(hs, 2)


@contextlib.contextmanager
def recurrent():
    """run learner_ref / qmix_ref with the recurrent agents' forward pass"""
    saved = lr.agents_forward
    lr.agents_forward = agents_forward
    try:
        yield
    finally:
        lr.agents_forward = saved


def dqn_update(st: lr.DqnState, batch, hp: lr.DqnHP):
    with recurrent():
        return lr.dqn_update(st, batch, hp)


def dqn_loss(theta, theta_tgt, agent_net, in_dim, out_dim, batch, hp, ret_ms=None):
    with recurrent():
        return lr.dqn_loss(theta, theta_tgt, agent_net, in_dim, out_dim, batch, hp, ret_ms)


def double_q_margin(st: lr.DqnState, batch, hp: lr.DqnHP):
    with recurrent():
        return lr.double_q_margin(st, batch, hp)


def dqn_kink_risk(st: lr.DqnState, batch, hp: lr.DqnHP):
    with recurrent():
        return lr.dqn_kink_risk(st, batch, hp)


def qmix_update(st: qr.QmixState, batch, hp: lr.DqnHP):
    with recurrent():
        return qr.qmix_update(st, batch, hp)


def qmix_kink_risk(st: qr.QmixState, batch, hp: lr.DqnHP):
    with recurrent():
        return qr.qmix_kink_risk(st, batch, hp)

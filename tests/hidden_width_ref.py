"""CPU restatement (PyTorch float32, autograd) of the agents' networks at a hidden width H of `layers: [H, H]` (1 <= H <= 128).  TEST
INFRASTRUCTURE ONLY.

oracle/learner_ref.py restates FCNetwork (utils/models.py:14-48) and oracle/gru_ref.py RNNNetwork (utils/models.py:51-116) at the shipped
layers = [128, 128].  This module restates the same two networks at width H, over flat parameter vectors in the compact device layout (the
reference's state_dict order per network: MLP P = H*in + H + H*H + H + out*H + out; GRU P = H*in + H + 6*H*H + 6*H + out*H + out), and runs
learner_ref's and qmix_ref's loss and update functions unchanged with them (`networks()`, the pattern of tests/gru_ac_ref.py), so every line of
loss arithmetic is shared with the 128-wide oracle.  Each call's width is read from the length of its flat vector (`width_of`).
"""
from __future__ import annotations

import contextlib
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import learner_ref as lr


# ---- parameter layouts --------------------------------------------------------------------------------------------------------------------------
def mlp_shapes(in_dim, out_dim, H):
    return ((H, in_dim), (H,), (H, H), (H,), (out_dim, H), (out_dim,))


def gru_shapes(in_dim, out_dim, H):
    return ((H, in_dim), (H,), (3 * H, H), (3 * H, H), (3 * H,), (3 * H,), (out_dim, H), (out_dim,))


def _shapes(recurrent):
    return gru_shapes if recurrent else mlp_shapes


def net_size(in_dim, out_dim, H, recurrent=False):
    return sum(int(np.prod(s)) for s in _shapes(recurrent)(in_dim, out_dim, H))


def split_net(flat, in_dim, out_dim, H, recurrent=False):
    """views of one network's flat parameters in state_dict order (MLP: w1, b1, w2, b2, w3, b3; GRU: the eight tensors of gru_ref.NAMES)"""
    out, o = [], 0
    for shape in _shapes(recurrent)(in_dim, out_dim, H):
        n = int(np.prod(shape))
        out.append(flat[o:o + n].view(*shape))
        o += n
    return out


def width_of(flat, agent_net, in_dim, out_dim, recurrent=False):
    """the hidden width H of the max(agent_net) + 1 networks of a flat vector, from its length (None: no width fits)"""
    P, rem = divmod(flat.numel(), max(agent_net) + 1)
    if rem or P <= out_dim:
        return None
    a, b = (6, in_dim + out_dim + 7) if recurrent else (1, in_dim + out_dim + 2)   # P = a H^2 + b H + out_dim
    H = int(round((math.sqrt(b * b + 4 * a * (P - out_dim)) - b) / (2 * a)))
    return H if H >= 1 and net_size(in_dim, out_dim, H, recurrent) == P else None


MLP_KEYS = ("network.0.weight", "network.0.bias", "network.2.weight", "network.2.bias", "network.4.weight", "network.4.bias")
GRU_KEYS = ("first_layer.weight", "first_layer.bias", "rnn.weight_ih_l0", "rnn.weight_hh_l0", "rnn.bias_ih_l0", "rnn.bias_hh_l0",
            "final_layer.weight", "final_layer.bias")


def state_dict_from_flat(flat, prefix, n_nets, in_dim, out_dim, H, recurrent=False):
    P, sd = net_size(in_dim, out_dim, H, recurrent), {}
    for k in range(n_nets):
        for name, t in zip(GRU_KEYS if recurrent else MLP_KEYS, split_net(flat[k * P:(k + 1) * P], in_dim, out_dim, H, recurrent)):
            sd[f"{prefix}.{k}.{name}"] = t.clone()
    return sd


def flat_from_state_dict(sd, prefix, n_nets, recurrent=False):
    return torch.cat([sd[f"{prefix}.{k}.{name}"].reshape(-1) for k in range(n_nets) for name in (GRU_KEYS if recurrent else MLP_KEYS)]).clone().float()


# ---- initialisation (the reference's rules and module order, so the RNG stream matches) ---------------------------------------------------------
def init_mlp(n_nets, in_dim, out_dim, H, orthogonal=True, generator=None):
    """utils/models.py:8-11,35-44: orthogonal(gain sqrt 2) weights + zero bias on every Linear (or nn.Linear default)."""
    parts = []
    for _ in range(n_nets):
        for (o, i) in ((H, in_dim), (H, H), (out_dim, H)):
            lin = torch.nn.Linear(i, o)
            if orthogonal:
                torch.nn.init.orthogonal_(lin.weight.data, gain=math.sqrt(2), generator=generator)
                torch.nn.init.constant_(lin.bias.data, 0)
            parts += [lin.weight.data.reshape(-1), lin.bias.data.reshape(-1)]
    return torch.cat(parts).float()


def init_gru(n_nets, in_dim, out_dim, H, orthogonal=True):
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


# ---- forward passes -----------------------------------------------------------------------------------------------------------------------------
def mlp(flat_net, x, in_dim, out_dim, H):
    w1, b1, w2, b2, w3, b3 = split_net(flat_net, in_dim, out_dim, H)
    z1 = F.linear(x, w1, b1); h1 = F.relu(z1)
    z2 = F.linear(h1, w2, b2); h2 = F.relu(z2)
    if lr._TAPS is not None and flat_net.requires_grad:   # learner_ref.kink_risk reads every ReLU of the differentiated passes
        h1.retain_grad(); h2.retain_grad()
        lr._TAPS.append((z1, h1, x)); lr._TAPS.append((z2, h2, h1))
    return F.linear(h2, w3, b3)


def gru_net(flat_net, x, in_dim, out_dim, H, h0=None):
    """x (L, B, in_dim) -> q (L, B, out_dim), h (L, B, H): every step's hidden state; h0 (B, H) or None = zeros."""
    w1, b1, wih, whh, bih, bhh, w3, b3 = split_net(flat_net, in_dim, out_dim, H, True)
    z1 = F.linear(x, w1, b1)
    x1 = F.relu(z1)
    if lr._TAPS is not None and flat_net.requires_grad:   # the first layer's ReLU is the net's only kink (oracle/gru_ref.py)
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


def agents_forward(flat, agent_net, xs, in_dim, out_dim, recurrent=False):
    """learner_ref.agents_forward at the width of `flat`: xs per agent; a GRU runs each sequence (L, B, D) from the zero state"""
    H = width_of(flat, agent_net, in_dim, out_dim, recurrent)
    assert H is not None, (flat.numel(), agent_net, in_dim, out_dim, recurrent)
    P = net_size(in_dim, out_dim, H, recurrent)
    if recurrent:
        return [gru_net(flat[k * P:(k + 1) * P], x, in_dim, out_dim, H)[0] for k, x in zip(agent_net, xs)]
    return [mlp(flat[k * P:(k + 1) * P], x, in_dim, out_dim, H) for k, x in zip(agent_net, xs)]


def act_steps(flat, agent_net, obs, in_dim, out_dim, h0=None):
    """model.act of recurrent networks over consecutive steps: obs (S, E, N, D), h0 (E, N, H) or None -> q (S, E, N, A), h (S, E, N, H)"""
    H = width_of(flat, agent_net, in_dim, out_dim, True)
    P = net_size(in_dim, out_dim, H, True)
    qs, hs = [], []
    for a, k in enumerate(agent_net):
        q, h = gru_net(flat[k * P:(k + 1) * P], obs[:, :, a], in_dim, out_dim, H, None if h0 is None else h0[:, a])
        qs.append(q); hs.append(h)
    return torch.stack(qs, 2), torch.stack(hs, 2)


@contextlib.contextmanager
def networks(recurrent=()):
    """run learner_ref / qmix_ref with this module's agents_forward; `recurrent`: the (in_dim, out_dim) pairs whose networks are GRUs (the actor
    and the critic of an actor-critic learner differ in out_dim; every other call is an MLP)"""
    saved = lr.agents_forward
    lr.agents_forward = lambda flat, agent_net, xs, in_dim, out_dim: agents_forward(flat, agent_net, xs, in_dim, out_dim, (in_dim, out_dim) in recurrent)
    try:
        yield
    finally:
        lr.agents_forward = saved

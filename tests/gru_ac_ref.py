"""CPU restatement (PyTorch float32, autograd) of the actor-critic learners with recurrent parts (actor.use_rnn / critic.use_rnn).  TEST
INFRASTRUCTURE ONLY.

Restated from (path:line in the reference project's marlbase/):
  utils/models.py:51-116     RNNNetwork (oracle/gru_ref.py restates it over flat parameters)
  ac/model.py:147-163        act / get_value carry the hiddens;  :189-246, 265-352 every update pass starts from hiddens=None (zeros)

learner_ref's A2C / PPO update, loss and ReLU-kink functions run unchanged with an agents_forward that picks the network kind of each call from the
flat vector's length: n_nets x P differs between the GRU and the MLP of the same widths.  So the actor and the critic are switched independently,
and the recurrent learners share every line of loss arithmetic with the feed-forward ones.  At a hidden width below 128 the networks are
tests/hidden_width_ref.py's, the width read from the vector's length as well.
"""
from __future__ import annotations

import contextlib

import torch

from oracle import gru_ref as gr
from oracle import learner_ref as lr
from tests import hidden_width_ref as hr


def is_recurrent(flat, agent_net, in_dim, out_dim):
    n_nets = max(agent_net) + 1
    if flat.numel() == n_nets * gr.net_size(in_dim, out_dim):
        return True
    if flat.numel() == n_nets * lr.net_size(in_dim, out_dim):
        return False
    # another hidden width (layers: [H, H], H < 128): the kind whose width fits the vector's length, which must be unambiguous
    rec, ff = hr.width_of(flat, agent_net, in_dim, out_dim, True), hr.width_of(flat, agent_net, in_dim, out_dim, False)
    assert (rec is None) != (ff is None), (flat.numel(), n_nets, in_dim, out_dim, rec, ff)
    return rec is not None


def agents_forward(flat, agent_net, xs, in_dim, out_dim):
    """learner_ref.agents_forward for either network kind at any width: xs per agent (L, P, D); a GRU runs each sequence from the zero state"""
    rec = is_recurrent(flat, agent_net, in_dim, out_dim)
    if rec and flat.numel() == (max(agent_net) + 1) * gr.net_size(in_dim, out_dim):
        return gr.agents_forward(flat, agent_net, xs, in_dim, out_dim)
    if not rec and flat.numel() == (max(agent_net) + 1) * lr.net_size(in_dim, out_dim):
        P = lr.net_size(in_dim, out_dim)
        return [lr.mlp(flat[k * P:(k + 1) * P], x, in_dim, out_dim) for k, x in zip(agent_net, xs)]
    return hr.agents_forward(flat, agent_net, xs, in_dim, out_dim, rec)


@contextlib.contextmanager
def mixed():
    """run learner_ref with this module's agents_forward"""
    saved = lr.agents_forward
    lr.agents_forward = agents_forward
    try:
        yield
    finally:
        lr.agents_forward = saved


def init_part(recurrent, n_nets, in_dim, out_dim):
    """one part's initial parameters by its own rule (global RNG): RNNNetwork's (orthogonal on final_layer only) or FCNetwork's"""
    return gr.init_flat(n_nets, in_dim, out_dim) if recurrent else lr.init_flat(n_nets, in_dim, out_dim)


def dqn_update(st: lr.DqnState, batch, hp: lr.DqnHP):
    """gru_ref's DQN functions for recurrent agents of any width"""
    with mixed():
        return lr.dqn_update(st, batch, hp)


def dqn_kink_risk(st: lr.DqnState, batch, hp: lr.DqnHP):
    with mixed():
        return lr.dqn_kink_risk(st, batch, hp)


def double_q_margin(st: lr.DqnState, batch, hp: lr.DqnHP):
    with mixed():
        return lr.double_q_margin(st, batch, hp)


def a2c_update(st: lr.A2CState, batch, hp: lr.A2CHP, step: int):
    with mixed():
        return lr.a2c_update(st, batch, hp, step)


def ppo_update(st: lr.A2CState, batch, hp: lr.A2CHP, step: int, num_epochs: int = 4, ppo_clip: float = 0.2):
    with mixed():
        return lr.ppo_update(st, batch, hp, step, num_epochs, ppo_clip)


def a2c_kink_risk(st: lr.A2CState, batch, hp: lr.A2CHP):
    with mixed():
        return lr.a2c_kink_risk(st, batch, hp)


def ppo_kink_risk(st: lr.A2CState, batch, hp: lr.A2CHP, res, ppo_clip, epoch=-1):
    with mixed():
        return lr.ppo_kink_risk(st, batch, hp, res, ppo_clip, epoch)


def act_steps(flat, agent_net, obs, in_dim, out_dim, h0=None):
    """act / get_value over consecutive steps of a recurrent part: obs (S, E, N, in_dim) -> outputs (S, E, N, out), h (S, E, N, H)"""
    if flat.numel() == (max(agent_net) + 1) * gr.net_size(in_dim, out_dim):
        return gr.act_steps(flat, agent_net, obs, in_dim, out_dim, h0)
    return hr.act_steps(flat, agent_net, obs, in_dim, out_dim, h0)


def joint(obs):
    """get_value's centralised inputs (ac/model.py:156-157): obs (..., N, D) -> (..., N, N * D), every agent reading all observations"""
    N = obs.shape[-2]
    j = obs.reshape(*obs.shape[:-2], N * obs.shape[-1])
    return j.unsqueeze(-2).expand(*obs.shape[:-2], N, j.shape[-1]).contiguous()


"""GPU: the wgmma forward path (3xTF32 split) against the FP32 FFMA forward kernel and the CPU oracle, dense
(model.act) and gathered (target-network pass) row sources, obs widths 15 / 27, outputs 6 / 1, ragged tiles, weight images freshly packed and
kept current by the optimiser step."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

from oracle import learner_ref as lr

pytestmark = pytest.mark.gpu


def _space(shape=None, n=None):
    return types.SimpleNamespace(shape=shape, n=n)


def _set_tc(on: bool):
    from codebase_b200 import _native as nat

    nat.check(nat.lib().marl_set_option(b"tensor_core_forward", C.c_int32(int(on))), "marl_set_option")


@pytest.fixture(autouse=True)
def _restore():
    yield
    _set_tc(True)


# updates: optimiser steps between the last full packing of the weight images and the forward.  0: images packed from the parameters; 3: images the
# Adam kernel rewrote parameter by parameter (pack_param, permuted K order), which every forward between two updates of a training run reads.
@pytest.mark.parametrize("updates", [3, 0])
@pytest.mark.parametrize("n_agents,D,sharing,E", [(2, 15, False, 4096), (2, 15, True, 1000), (4, 27, False, 333), (3, 32, [0, 1, 0], 129), (2, 15, False, 1),
                                                  (2, 15, False, 40000), (1, 9, False, 20000)])   # the last two: several tiles per CTA
def test_dense_forward_tc_vs_ffma_vs_oracle(n_agents, D, sharing, E, updates):
    from codebase_b200.dqn.model import QNetwork
    from codebase_b200.lbf import TrajStore

    rng = np.random.default_rng(E)
    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=1.0, double_q=True, target_update_interval_or_tau=200, standardise_returns=False)
    T, cap, B = 25, 16, 8
    m = QNetwork([_space(shape=(D,))] * n_agents, [_space(n=6)] * n_agents, cfg, [128, 128], sharing, False, True, "cuda", max_batch=B, max_episode_length=T)
    m.theta.mul_(1.7)  # not the orthogonal-init special case
    m.theta.add_(torch.as_tensor(0.01 * rng.standard_normal(m.theta.numel()), dtype=torch.float32).to(m.theta.device).view_as(m.theta))
    m.params_changed()  # direct writes
    obs = torch.tensor(rng.integers(-1, 15, size=(E, n_agents, D)).astype(np.float32), device="cuda")
    _set_tc(True)
    if updates:
        ts = TrajStore(cap, n_agents, T, D, m.device)
        ts.obs.copy_(torch.as_tensor(rng.integers(-1, 15, size=(cap, n_agents, T + 1, D)).astype(np.float32)))
        ts.act.copy_(torch.as_tensor(rng.integers(0, 6, size=(cap, n_agents, T)).astype(np.int32)))
        ts.rew.copy_(torch.as_tensor(rng.random((cap, n_agents, T)).astype(np.float32)))
        ts.filled.fill_(1)
        ts.done[:, T] = 1
        before = m.theta.clone()
        for _ in range(updates):
            m.update_from_store(ts, torch.as_tensor(rng.integers(0, cap, size=B).astype(np.int32), device="cuda"))
        assert not torch.equal(before, m.theta)
    q_tc = m.q_values(obs).cpu().numpy()
    q_tc2 = m.q_values(obs).cpu().numpy()
    assert np.array_equal(q_tc, q_tc2), "the tensor-core forward is not deterministic"
    _set_tc(False)
    q_ff = m.q_values(obs).cpu().numpy()
    want = torch.stack(lr.agents_forward(m.theta.cpu(), m.agent_net, [obs[:, i].cpu() for i in range(n_agents)], D, 6), 1).numpy()
    scale = max(1.0, float(np.abs(want).max()))
    assert np.abs(q_ff - want).max() / scale < 1e-5
    assert np.abs(q_tc - want).max() / scale < 1e-5, np.abs(q_tc - want).max()
    assert np.abs(q_tc - q_ff).max() / scale < 1e-5


def test_a2c_value_and_logit_passes_on_tensor_cores():
    from codebase_b200.ac.model import A2CNetwork

    rng = np.random.default_rng(0)
    hp = lr.A2CHP()
    cfg = types.SimpleNamespace(optimizer="Adam", lr=hp.lr, gamma=hp.gamma, grad_clip=hp.grad_clip, n_steps=hp.n_steps, entropy_coef=hp.entropy_coef,
                                value_loss_coef=hp.value_loss_coef, target_update_interval_or_tau=hp.target_update_interval_or_tau, standardise_returns=False)
    net = types.SimpleNamespace(layers=[128, 128], parameter_sharing=False, use_rnn=False, use_orthogonal_init=True, centralised=False)
    m = A2CNetwork([_space(shape=(15,))] * 2, [_space(n=6)] * 2, cfg, net, net, "cuda", max_envs=700, max_episode_length=25)
    obs = torch.tensor(rng.integers(-1, 8, size=(700, 2, 15)).astype(np.float32), device="cuda")
    outs = {}
    for on in (True, False):
        _set_tc(on)
        outs[on] = (m.logits(obs).cpu().numpy(), m.values(obs).cpu().numpy(), m.values(obs, target=True).cpu().numpy())
    for a, b in zip(outs[True], outs[False]):
        assert np.abs(a - b).max() < 1e-5 * max(1.0, np.abs(b).max())

"""λ-returns (algorithm.gae_lambda) on the CPU: the oracle's mixture of n-step returns against the hand-written recursion and against the
reference's n-step returns at its two ends, the oracle's A2C / PPO updates at λ = 0 and λ = 1 against the reference's own A2CNetwork / PPONetwork
at n_steps = 1 and n_steps = T (tests/golden/gae_reference.npz), and the configuration: the four actor-critic configs carry the option, and a value
that is not a number in [0, 1] is refused before any native call."""
import copy
import types

import numpy as np
import pytest
import torch

from oracle import learner_ref as lr
from tests import gae_ref as gr
from tests.helpers import STRIDE, ac_oracle_batch, reference_outputs, space


def _sequences(rng, T, B=6, N=3):
    """rewards (T, B, N), dones (T+1, B, N) with episodes that end before T (and some that run to T unterminated), values (T+1, B, N)"""
    rew = rng.standard_normal((T, B, N))
    done = np.zeros((T + 1, B, N))
    for b in range(B):
        end = int(rng.integers(1, T + 1))
        if end < T or rng.random() < 0.5:
            done[end, b] = 1.0
    return rew, done, rng.standard_normal((T + 1, B, N))


@pytest.mark.parametrize("T", [1, 2, 7, 33])
@pytest.mark.parametrize("lam", [0.0, 0.3, 0.95, 1.0])
@pytest.mark.parametrize("gamma", [0.9, 0.99])
def test_mixture_equals_the_recursion(T, lam, gamma):
    rew, done, v = _sequences(np.random.default_rng(T * 100 + int(lam * 10)), T)
    want = gr.recursion(rew, done, v, lam, gamma)
    got = gr.lambda_returns(rew, done, v, lam, gamma)
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("T", [1, 5, 26])
def test_mixture_ends_are_the_reference_nstep_returns(T):
    """λ = 0 is compute_nstep_returns with n_steps = 1, λ = 1 with n_steps = T (no bootstrap: the return to the end of the stored episode); every
    G^(n) of the mixture is compute_nstep_returns with n_steps = n"""
    rew, done, v = _sequences(np.random.default_rng(T), T)
    t = lambda x: torch.tensor(x, dtype=torch.float64)   # noqa: E731
    G = gr.nstep_all(rew, done, v, 0.97)
    for n in range(1, T + 1):
        np.testing.assert_allclose(G[n - 1], lr.nstep_returns(t(rew), t(done), t(v), n, 0.97).numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(gr.lambda_returns(rew, done, v, 0.0, 0.97), lr.nstep_returns(t(rew), t(done), t(v), 1, 0.97).numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(gr.lambda_returns(rew, done, v, 1.0, 0.97), lr.nstep_returns(t(rew), t(done), t(v), T, 0.97).numpy(), rtol=1e-12, atol=1e-12)


def _close(a, b, tol=1e-5):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert np.allclose(a, b, rtol=tol, atol=tol), float(np.abs(a - b).max())


@pytest.mark.parametrize("key", list(gr.GOLDEN_CASES))
def test_oracle_lambda_ends_match_the_reference(key):
    """the oracle's updates with λ-returns at λ = 0 (resp. 1) -- and n_steps = 5, which the λ-returns do not read -- against what the reference's
    A2CNetwork / PPONetwork computed with n_steps = 1 (resp. T): first returns, losses, running statistics, parameters"""
    g = reference_outputs("gae_reference")
    cls, _, _, _, steps, epochs, clip, _, _, std, _, lam = gr.GOLDEN_CASES[key]
    st = gr.golden_state(key)
    hp = lr.A2CHP(grad_clip=float(clip or 0.0), target_update_interval_or_tau=2, n_steps=5)
    metrics = []
    with gr.lambda_returns_in(lam):
        for u, (step, s) in enumerate(zip(steps, gr.golden_batches(key))):
            b = ac_oracle_batch(s)
            if u == 0:
                with torch.no_grad():   # the returns before the running statistics absorb them
                    obs = list(torch.split(b["obss"], gr.D, dim=-1))
                    cobs, CD = st.critic_inputs(obs)
                    nv = torch.cat(lr.agents_forward(st.target, st.critic_net, cobs, CD, 1), dim=-1)
                    done = b["dones"].unsqueeze(-1).repeat(1, 1, gr.N)
                    _close(lr.nstep_returns(b["rewards"], done, nv, hp.n_steps, hp.gamma), g[f"{key}_returns0"])
            got = lr.ppo_update(st, b, hp, step, epochs, 0.2) if cls == "PPONetwork" else lr.a2c_update(st, b, hp, step)
            metrics.append([got[k] for k in gr.GOLDEN_METRICS])
    _close(metrics, g[f"{key}_metrics"])
    if std:
        _close(st.ret_ms.mean.numpy(), g[f"{key}_ret_mean"]); _close(st.ret_ms.var.numpy(), g[f"{key}_ret_var"])
        assert abs(st.ret_ms.count - float(g[f"{key}_ret_count"])) < 1e-9
    for mine, name in ((st.actor, "actor"), (st.critic, "critic"), (st.target, "target")):
        d = np.abs(mine.numpy()[::STRIDE] - g[f"{key}_{name}"])
        assert np.quantile(d, 0.999) < 1e-5, (name, d.max())


def test_lambda_returns_in_restores_the_nstep_returns():
    saved = lr.nstep_returns
    with gr.lambda_returns_in(0.5):
        assert lr.nstep_returns is not saved
    assert lr.nstep_returns is saved
    with gr.lambda_returns_in(None):
        assert lr.nstep_returns is saved


# ---- configuration -------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alg", ["ia2c", "ippo", "maa2c", "mappo"])
def test_configs_carry_gae_lambda(alg):
    from codebase_b200 import config

    base = [f"+algorithm={alg}", "env.name=lbforaging:Foraging-8x8-2p-3f-v3", "env.time_limit=25"]
    assert config.compose(base).algorithm.gae_lambda is None
    assert config.compose(base + ["algorithm.gae_lambda=0.95"]).algorithm.gae_lambda == 0.95
    assert config.compose(base + ["algorithm.gae_lambda=1"]).algorithm.gae_lambda == 1


@pytest.mark.parametrize("value,want", [(None, None), (0, 0.0), (0.95, 0.95), (1, 1.0), (np.float32(0.5), 0.5)])
def test_gae_lambda_parsing(value, want):
    from codebase_b200.ac.model import gae_lambda

    assert gae_lambda(types.SimpleNamespace(gae_lambda=value)) == want
    assert gae_lambda(types.SimpleNamespace()) is None


BAD = [-0.01, 1.0001, float("nan"), float("inf"), "0.95", True, [0.9]]


@pytest.mark.parametrize("value", BAD)
@pytest.mark.parametrize("cls", ["A2CNetwork", "PPONetwork"])
def test_bad_gae_lambda_is_refused_before_any_native_call(value, cls, monkeypatch):
    from codebase_b200 import _native as nat
    from codebase_b200.ac import model as M

    def no_native(*a, **k):
        raise AssertionError("a native call was made")

    monkeypatch.setattr(nat, "lib", no_native)
    monkeypatch.setattr(torch.cuda, "is_available", no_native)
    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=False, n_steps=5, entropy_coef=0.001, value_loss_coef=0.5,
                                target_update_interval_or_tau=200, standardise_returns=False, num_epochs=4, ppo_clip=0.2, gae_lambda=value)
    net = types.SimpleNamespace(layers=[128, 128], parameter_sharing=False, use_rnn=False, use_orthogonal_init=True, centralised=False)
    with pytest.raises(ValueError, match="gae_lambda"):
        getattr(M, cls)([space(shape=(15,))] * 2, [space(n=6)] * 2, cfg, net, copy.copy(net), "cuda")

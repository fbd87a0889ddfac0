"""TD(λ) targets of IDQN, VDN and QMIX (algorithm.td_lambda) on the CPU: the recursion against the explicit mixture of n-step returns, its two ends
(λ = 0: the one-step target; λ = 1: the discounted return to the end of the filled episode, bootstrapped there), the cut at unfilled rows, the
float64 oracle losses at λ = 0 against the reference's losses (oracle.learner_ref.dqn_loss, tests/qmix_options_ref.qmix_loss, which the goldens
pin), and the configuration: the option's place in idqn / vdn / qmix, its parsing, and its refusals before and at the native call."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

from oracle import learner_ref as lr
from oracle import qmix_ref as qr
from tests import qmix_options_ref as qo
from tests import td_lambda_ref as tl
from tests.helpers import space


def _sequences(rng, T, M=7, stale_filled=True):
    """rewards, dones (T+1), filled, bootstrap values of M sequences: ragged episodes (done before T, unterminated ones, unfilled tails) and, with
    stale_filled, rows marked filled again after an unfilled gap (a re-used replay slot's stale tail)"""
    rew, boot = rng.standard_normal((T, M)), rng.standard_normal((T, M))
    done, filled = np.zeros((T + 1, M)), np.zeros((T, M))
    for m in range(M):
        L = int(rng.integers(1, T + 1))
        filled[:L, m] = 1.0
        if L < T or rng.random() < 0.5:
            done[L, m] = float(rng.random() < 0.7)
        if stale_filled and L + 1 < T and m % 2:
            filled[L + 1:, m] = 1.0
            done[L + 1:, m] = rng.random(T - L) < 0.2
    return rew, done, filled, boot


def _G(rew, done, filled, boot, lam, gamma):
    t = lambda x: torch.tensor(x, dtype=torch.float64)   # noqa: E731
    return tl.lambda_targets(t(rew), t(done), t(filled), t(boot), lam, gamma).numpy()


@pytest.mark.parametrize("T", [1, 2, 7, 33])
@pytest.mark.parametrize("lam", [0.0, 0.3, 0.6, 1.0])
@pytest.mark.parametrize("gamma", [0.9, 0.99])
def test_recursion_equals_the_mixture_of_nstep_returns(T, lam, gamma):
    rew, done, filled, boot = _sequences(np.random.default_rng(T * 100 + int(lam * 10)), T)
    np.testing.assert_allclose(_G(rew, done, filled, boot, lam, gamma), tl.lambda_mixture(rew, done, filled, boot, lam, gamma), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("T", [1, 4, 26])
def test_lambda_zero_is_the_one_step_target(T):
    rew, done, filled, boot = _sequences(np.random.default_rng(T), T)
    np.testing.assert_allclose(_G(rew, done, filled, boot, 0.0, 0.97), rew + 0.97 * (1.0 - done[1:]) * boot, rtol=1e-15, atol=1e-15)


@pytest.mark.parametrize("T", [1, 4, 26])
def test_lambda_one_is_the_discounted_return_of_the_filled_episode(T):
    """λ = 1: Σ_k γ^k c_k r_{t+k} up to the last filled step t + L - 1, plus γ^L c_L v_{t+L}"""
    rew, done, filled, boot = _sequences(np.random.default_rng(T + 5), T)
    want = np.zeros_like(rew)
    for m in range(rew.shape[1]):
        for t in range(T):
            L = 1
            while t + L < T and filled[t + L, m] > 0:
                L += 1
            c, acc = 1.0, 0.0
            for k in range(L):
                acc += 0.95 ** k * c * rew[t + k, m]
                c *= 1.0 - done[t + k + 1, m]
            want[t, m] = acc + 0.95 ** L * c * boot[t + L - 1, m]
    np.testing.assert_allclose(_G(rew, done, filled, boot, 1.0, 0.95), want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("lam", [0.6, 1.0])
def test_stale_rows_never_reach_a_filled_rows_target(lam):
    """rows after the first unfilled row following t (rewards, dones, bootstrap values, even rows marked filled again) leave G_t unchanged"""
    T, rng = 30, np.random.default_rng(3)
    rew, done, filled, boot = _sequences(rng, T, M=1, stale_filled=False)
    filled[:] = 0.0; done[:] = 0.0
    filled[:12] = 1.0                      # filled rows 0..11, row 12 unfilled (truncated: no done), then a stale tail
    filled[14:] = 1.0
    G = _G(rew, done, filled, boot, lam, 0.99)
    rew2, done2, boot2 = rew.copy(), done.copy(), boot.copy()
    rew2[12:] = rng.standard_normal((T - 12, 1)); done2[13:] = 1.0; boot2[12:] = rng.standard_normal((T - 12, 1))
    G2 = _G(rew2, done2, filled, boot2, lam, 0.99)
    np.testing.assert_array_equal(G2[:12], G[:12])
    assert not np.allclose(G2[12:], G[12:])


# ---- the oracle losses at λ = 0: the reference's own --------------------------------------------------------------------------------------------
def _dqn_case(mixer, seed, N=3, D=5, A=4, T=9, B=6):
    g = torch.Generator().manual_seed(seed)
    theta, theta_tgt = lr.init_flat(N, D, A, generator=g), lr.init_flat(N, D, A, generator=g)
    batch = qr.random_batch(N, T, B, D, A, seed=seed, ragged=True)
    if mixer == 0:
        batch["rewards"] = torch.randn(N, T, B, generator=g)
    return theta, theta_tgt, list(range(N)), D, A, batch


@pytest.mark.parametrize("mixer", [0, 1])
@pytest.mark.parametrize("double_q", [True, False])
@pytest.mark.parametrize("standardise", [False, True])
def test_oracle_dqn_loss_at_lambda_zero_is_the_reference_loss(mixer, double_q, standardise):
    theta, theta_tgt, nets, D, A, batch = _dqn_case(mixer, 11 + mixer)
    hp = lr.DqnHP(double_q=double_q, mixer=mixer)
    b64 = {k: (v if k == "actions" else v.double()) for k, v in batch.items()}
    shape = (1,) if mixer == 1 else (len(nets),)
    ms_a, ms_b = (lr.RunningMeanStdRef(shape), lr.RunningMeanStdRef(shape)) if standardise else (None, None)
    want = lr.dqn_loss(theta.double(), theta_tgt.double(), nets, D, A, b64, hp, ret_ms=ms_a)
    got = tl.dqn_loss(theta, theta_tgt, nets, D, A, batch, hp, ret_ms=ms_b, lam=0.0)
    tol = 1e-6 if standardise else 1e-12   # the statistics absorb the float32 returns here, the float64 ones there
    assert abs(float(got) - float(want)) <= tol * max(1.0, abs(float(want)))
    with tl.td_lambda_in(0.0):
        st = lr.DqnState(theta.clone(), theta_tgt.clone(), nets, D, A, ret_ms=lr.RunningMeanStdRef(shape) if standardise else None)
        res = lr.dqn_update(st, batch, hp)
    st0 = lr.DqnState(theta.clone(), theta_tgt.clone(), nets, D, A, ret_ms=lr.RunningMeanStdRef(shape) if standardise else None)
    ref = lr.dqn_update(st0, batch, hp)
    assert abs(res["loss"] - ref["loss"]) <= 1e-5 * max(1.0, abs(ref["loss"]))
    np.testing.assert_allclose(res["grad"].numpy(), ref["grad"].numpy(), rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize("hl", [1, 2])
@pytest.mark.parametrize("standardise", [False, True])
def test_oracle_qmix_loss_at_lambda_zero_is_the_reference_loss(hl, standardise):
    N, D, A, T, B, E = 3, 5, 4, 8, 6, 16
    torch.manual_seed(5)
    theta, theta_tgt = lr.init_flat(N, D, A), lr.init_flat(N, D, A)
    mix = qo.init_mixer_flat(N, N * D, E, 32, hl)
    st = lambda: qo.QmixOptState(theta.clone(), theta_tgt.clone(), mix.clone(), mix.clone() + 0.01, list(range(N)), D, A, embed_dim=E,   # noqa: E731
                                 hypernet_layers=hl, ret_ms=lr.RunningMeanStdRef((1,)) if standardise else None)
    batch = qr.random_batch(N, T, B, D, A, seed=9, ragged=True)
    b64 = {k: (v if k == "actions" else v.double()) for k, v in batch.items()}
    hp = lr.DqnHP()
    sa, sb = st(), st()
    sa.theta_tgt, sa.mix_tgt = sa.theta_tgt.double(), sa.mix_tgt.double()
    want = qo.qmix_loss(theta.double(), mix.double(), sa, b64, hp)
    got = tl.qmix_loss(theta, mix, sb, batch, hp, lam=0.0)
    tol = 1e-6 if standardise else 1e-12
    assert abs(float(got) - float(want)) <= tol * max(1.0, abs(float(want)))


def test_td_lambda_in_restores_the_one_step_losses():
    saved = lr.dqn_loss, qr.qmix_loss
    with tl.td_lambda_in(0.5):
        assert lr.dqn_loss is not saved[0] and qr.qmix_loss is not saved[1]
    assert (lr.dqn_loss, qr.qmix_loss) == saved
    with tl.td_lambda_in(None):
        assert (lr.dqn_loss, qr.qmix_loss) == saved


# ---- configuration -------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alg", ["idqn", "vdn", "qmix"])
def test_configs_carry_td_lambda(alg):
    from codebase_b200 import config

    base = [f"+algorithm={alg}", "env.name=lbforaging:Foraging-8x8-2p-3f-v3", "env.time_limit=25"]
    assert config.compose(base).algorithm.td_lambda is None
    assert config.compose(base + ["algorithm.td_lambda=0.6"]).algorithm.td_lambda == 0.6
    assert config.compose(base + ["algorithm.td_lambda=1"]).algorithm.td_lambda == 1


@pytest.mark.parametrize("value,want", [(None, None), (0, 0.0), (0.6, 0.6), (1, 1.0), (np.float32(0.5), 0.5)])
def test_td_lambda_parsing(value, want):
    from codebase_b200.dqn.model import td_lambda

    assert td_lambda(types.SimpleNamespace(td_lambda=value)) == want
    assert td_lambda(types.SimpleNamespace()) is None


BAD = [-0.01, 1.0001, float("nan"), float("inf"), "0.6", True, [0.6]]


@pytest.mark.parametrize("value", BAD)
@pytest.mark.parametrize("cls", ["QNetwork", "VDNetwork", "QMixNetwork"])
def test_bad_td_lambda_is_refused_before_any_native_call(value, cls, monkeypatch):
    from codebase_b200 import _native as nat
    from codebase_b200.dqn import model as M

    def no_native(*a, **k):
        raise AssertionError("a native call was made")

    monkeypatch.setattr(nat, "lib", no_native)
    monkeypatch.setattr(torch.cuda, "is_available", no_native)
    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=1.0, double_q=True, target_update_interval_or_tau=200,
                                standardise_returns=False, td_lambda=value)
    args = ([space(shape=(15,))] * 2, [space(n=6)] * 2, cfg, [128, 128], False, False, True)
    with pytest.raises(ValueError, match="td_lambda"):
        if cls == "QMixNetwork":
            M.QMixNetwork(*args, dict(embed_dim=64, hypernet_layers=2, hypernet_embed=32), "cuda")
        else:
            getattr(M, cls)(*args, "cuda")


@pytest.mark.parametrize("lam", [-0.5, 1.5, float("nan"), float("inf")])
def test_native_entry_point_refuses_lambda_outside_0_1(lam):
    """the C ABI refuses the value itself (checked before the handle, so no device is needed to see it)"""
    from codebase_b200 import _native as nat

    lib = nat.lib()
    rc = lib.marl_dqn_set_td_lambda(None, C.c_int32(1), C.c_float(lam))
    assert rc < 0 and b"outside [0, 1]" in lib.marl_last_error()
    rc = lib.marl_dqn_set_td_lambda(None, C.c_int32(1), C.c_float(0.6))   # a valid λ gets as far as the handle
    assert rc < 0 and b"NULL handle" in lib.marl_last_error()

"""The Huber TD loss of IDQN, VDN and QMIX (algorithm.huber_delta) on the CPU: the float64 oracle (tests/huber_ref.py) against the reference's own
learners with mse_loss replaced by huber_loss (tests/golden/huber_reference.npz, from tests/golden/make_huber_golden.py) with TD errors on both
sides of delta; the large-delta limit, half the reference's squared-error loss and gradient (oracle.learner_ref.dqn_loss and
tests/qmix_options_ref.qmix_loss, which the goldens pin); and the configuration: the option's place in idqn / vdn / qmix, its parsing, and its
refusals before and at the native call."""
import copy
import ctypes as C
import types

import numpy as np
import pytest
import torch

from oracle import learner_ref as lr
from oracle import qmix_ref as qr
from tests import huber_ref as hr
from tests import qmix_options_ref as qo
from tests.helpers import STRIDE, reference_outputs, space


def test_huber_is_torchs_huber_loss():
    d = torch.linspace(-3.0, 3.0, 601, dtype=torch.float64)
    for delta in (0.1, 1.0, 2.5):
        want = torch.nn.functional.huber_loss(d, torch.zeros_like(d), reduction="none", delta=delta)
        torch.testing.assert_close(hr.huber(d, delta), want, rtol=1e-15, atol=1e-15)


@pytest.mark.parametrize("name", list(hr.GOLDEN_CASES))
def test_oracle_matches_reference(name):
    """three updates of the reference's learner with huber_loss from the same weights and batches: the loss of every update, the first update's
    gradient, the parameters after the last; the first batch has TD errors inside and outside the band"""
    g, c = reference_outputs("huber_reference"), hr.GOLDEN_CASES[name]
    st, hp = hr.golden_state(c), hr.golden_hp(c)
    for u, batch in enumerate(hr.golden_batches(c)):
        if u == 0:
            inside, outside = hr.branches(hr.golden_td(c, st, batch, hp), batch["filled"], c.delta)
            assert inside >= 10 and outside >= 10, (inside, outside)
        got = hr.golden_update(c, st, batch, hp)
        want = float(g[f"{name}_loss"][u])
        assert abs(got["loss"] - want) <= 1e-5 * max(1.0, abs(want)), f"loss of update {u}: {got['loss']} vs {want}"
        if u == 0:
            grads = [("grad", "grad0")] + ([("mix_grad", "mix_grad0")] if c.cls == "QMixNetwork" else [])
            for mine, key in grads:
                ref = g[f"{name}_{key}"]
                err = float(np.abs(got[mine].numpy()[::STRIDE] - ref).max())
                assert err <= 1e-5 * max(1e-3, float(np.abs(ref).max())), f"{key}: {err:.3e}"
    mine = [(st.theta, "theta"), (st.theta_tgt, "theta_tgt")]
    if c.cls == "QMixNetwork":
        mine += [(st.mix, "mix"), (st.mix_tgt, "mix_tgt")]
    for t, key in mine:
        assert np.quantile(np.abs(t.numpy()[::STRIDE] - g[f"{name}_{key}"]), 0.999) < 1e-5, key


@pytest.mark.parametrize("name", list(hr.GOLDEN_CASES))
def test_a_different_delta_misses_the_reference(name):
    """the fixture pins delta: the same updates with twice the case's delta do not reproduce it"""
    g, c = reference_outputs("huber_reference"), hr.GOLDEN_CASES[name]
    st, hp = hr.golden_state(c), hr.golden_hp(c)
    got = hr.golden_update(c, st, hr.golden_batches(c)[0], hp, delta=2 * c.delta)
    assert abs(got["loss"] - float(g[f"{name}_loss"][0])) > 1e-3


# ---- the large-delta limit: half the reference's squared error -------------------------------------------------------------------------------------
def _half(got, want):
    """got = want / 2 to 1e-5 of the gradient's scale (the squared-error oracles run in float32)"""
    err = float((got.double() - 0.5 * want.double()).abs().max())
    assert err <= 1e-5 * float(want.abs().max()), err


@pytest.mark.parametrize("mixer", [0, 1])
@pytest.mark.parametrize("double_q", [True, False])
@pytest.mark.parametrize("standardise", [False, True])
def test_large_delta_is_half_the_squared_error(mixer, double_q, standardise):
    N, D, A, T, B = 3, 5, 4, 9, 6
    g = torch.Generator().manual_seed(17 + mixer)
    theta, theta_tgt = lr.init_flat(N, D, A, generator=g), lr.init_flat(N, D, A, generator=g)
    batch = qr.random_batch(N, T, B, D, A, seed=3 + mixer, ragged=True)
    batch["rewards"] = 3.0 * torch.randn(N, T, B, generator=g)
    hp = lr.DqnHP(double_q=double_q, mixer=mixer)
    shape = (1,) if mixer == 1 else (N,)
    ms = (lambda: lr.RunningMeanStdRef(shape)) if standardise else (lambda: None)
    nets = list(range(N))
    st_h, st_m = lr.DqnState(theta.clone(), theta_tgt.clone(), nets, D, A, ret_ms=ms()), lr.DqnState(theta.clone(), theta_tgt.clone(), nets, D, A, ret_ms=ms())
    with hr.huber_in(1e6):
        got = lr.dqn_update(st_h, batch, hp)
    want = lr.dqn_update(st_m, batch, hp)
    tol = 1e-5 if standardise else 1e-6   # the statistics absorb float32 returns there, float64 ones in the reference's oracle
    assert abs(got["loss"] - 0.5 * want["loss"]) <= tol * max(1.0, abs(want["loss"]))
    _half(got["grad"], want["grad"])


@pytest.mark.parametrize("hl", [1, 2])
def test_large_delta_is_half_the_squared_error_qmix(hl):
    N, D, A, T, B = 3, 5, 4, 8, 6
    torch.manual_seed(7 + hl)
    theta, theta_tgt = lr.init_flat(N, D, A), lr.init_flat(N, D, A)
    mix = qo.init_mixer_flat(N, N * D, 64, 32, hl)
    st = qo.QmixOptState(theta, theta_tgt, mix, mix + 0.01, list(range(N)), D, A, hypernet_layers=hl)
    batch = qr.random_batch(N, T, B, D, A, seed=9, ragged=True)
    batch["rewards"][:] = 3.0 * torch.randn(1, T, B)
    hp = lr.DqnHP()
    st_h, st_m = copy.deepcopy(st), copy.deepcopy(st)
    with hr.huber_in(1e6):
        got = qr.qmix_update(st_h, batch, hp)
    want = qo.qmix_update(st_m, batch, hp)
    assert abs(got["loss"] - 0.5 * want["loss"]) <= 1e-6 * max(1.0, abs(want["loss"]))
    for k in ("grad", "mix_grad"):
        _half(got[k], want[k])


def test_huber_in_restores_the_squared_error():
    saved = lr.dqn_loss, qr.qmix_loss
    with hr.huber_in(0.5, lam=0.6):
        assert lr.dqn_loss is not saved[0] and qr.qmix_loss is not saved[1]
    assert (lr.dqn_loss, qr.qmix_loss) == saved
    with hr.huber_in(None):
        assert (lr.dqn_loss, qr.qmix_loss) == saved


# ---- configuration -------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alg", ["idqn", "vdn", "qmix"])
def test_configs_carry_huber_delta(alg):
    from codebase_b200 import config

    base = [f"+algorithm={alg}", "env.name=lbforaging:Foraging-8x8-2p-3f-v3", "env.time_limit=25"]
    assert config.compose(base).algorithm.huber_delta is None
    assert config.compose(base + ["algorithm.huber_delta=1.0"]).algorithm.huber_delta == 1.0
    assert config.compose(base + ["algorithm.huber_delta=10"]).algorithm.huber_delta == 10


@pytest.mark.parametrize("value,want", [(None, None), (1, 1.0), (0.25, 0.25), (1e4, 1e4), (np.float32(0.5), 0.5)])
def test_huber_delta_parsing(value, want):
    from codebase_b200.dqn.model import huber_delta

    assert huber_delta(types.SimpleNamespace(huber_delta=value)) == want
    assert huber_delta(types.SimpleNamespace()) is None


BAD = [0, 0.0, -1.0, float("nan"), float("inf"), float("-inf"), "1.0", True, [1.0]]


@pytest.mark.parametrize("value", BAD)
@pytest.mark.parametrize("cls", ["QNetwork", "VDNetwork", "QMixNetwork"])
def test_bad_huber_delta_is_refused_before_any_native_call(value, cls, monkeypatch):
    from codebase_b200 import _native as nat
    from codebase_b200.dqn import model as M

    def no_native(*a, **k):
        raise AssertionError("a native call was made")

    monkeypatch.setattr(nat, "lib", no_native)
    monkeypatch.setattr(torch.cuda, "is_available", no_native)
    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=1.0, double_q=True, target_update_interval_or_tau=200,
                                standardise_returns=False, td_lambda=None, huber_delta=value)
    args = ([space(shape=(15,))] * 2, [space(n=6)] * 2, cfg, [128, 128], False, False, True)
    with pytest.raises(ValueError, match="huber_delta"):
        if cls == "QMixNetwork":
            M.QMixNetwork(*args, dict(embed_dim=64, hypernet_layers=2, hypernet_embed=32), "cuda")
        else:
            getattr(M, cls)(*args, "cuda")


@pytest.mark.parametrize("delta", [0.0, -0.5, float("nan"), float("inf")])
def test_native_entry_point_refuses_a_bad_delta(delta):
    """the C ABI refuses the value itself (checked before the handle, so no device is needed to see it)"""
    from codebase_b200 import _native as nat

    lib = nat.lib()
    rc = lib.marl_dqn_set_huber_delta(None, C.c_int32(1), C.c_float(delta))
    assert rc < 0 and b"finite number > 0" in lib.marl_last_error()
    rc = lib.marl_dqn_set_huber_delta(None, C.c_int32(1), C.c_float(1.0))   # a valid delta gets as far as the handle
    assert rc < 0 and b"NULL handle" in lib.marl_last_error()
    rc = lib.marl_dqn_set_huber_delta(None, C.c_int32(0), C.c_float(delta))   # switching off takes no delta
    assert rc < 0 and b"NULL handle" in lib.marl_last_error()

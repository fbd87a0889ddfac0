"""QMIX's two remaining reference options (marlbase/dqn/model.py:272-443): one-layer hypernetworks (`mixing.hypernet_layers=1`) and
`standardise_returns`.  CPU: the oracle restatement against outputs of the reference's own QMixNetwork (tests/golden/qmix_options_reference.npz),
the weight-gradient decompositions of the one-layer mixer, and the refusal of other hypernetwork depths.  The CUDA path is checked in
tests/test_qmix_options_gpu.py.  The oracle is tests/qmix_options_ref.py (oracle/qmix_ref.py's update with either mixer and the standardisation).
The fixture regenerates with  MARL_REFERENCE_ROOT=<checkout> python -m tests.test_qmix_options"""
import ctypes as C
import os
import types
from dataclasses import dataclass

import numpy as np
import pytest
import torch

from oracle import learner_ref as lr
from oracle import qmix_ref as qr
from tests import qmix_options_ref as qo
from tests.helpers import STRIDE, load_params, reference_outputs, seeded_params

A, T, B = 6, 6, 16
GOLDEN_DIR = os.path.join(os.path.dirname(__file__), "golden")


@dataclass(frozen=True)
class Case:
    hl: int                     # mixing.hypernet_layers
    standardise: bool = False
    tu: float = 2.0             # target_update_interval_or_tau
    sharing: bool = False
    N: int = 2
    D: int = 9
    B: int = B
    seed: int = 31


CASES = {
    "h1_hard": Case(hl=1),
    "h1_std_polyak": Case(hl=1, standardise=True, tu=0.05, seed=32),
    "h2_std_shared": Case(hl=2, standardise=True, sharing=True, seed=33),
    "h1_n4_d27": Case(hl=1, N=4, D=27, B=8, seed=34),
}


def batch(rng, c: Case):
    """(N, T+1, B, D) observations, team rewards, a few terminal steps and unfilled rows (the layout of tests/test_qmix.py)"""
    rew = np.repeat(rng.random((1, T, c.B)), c.N, axis=0)
    return dict(obss=torch.tensor(rng.standard_normal((c.N, T + 1, c.B, c.D)), dtype=torch.float32), actions=torch.tensor(rng.integers(0, A, (c.N, T, c.B))),
                rewards=torch.tensor(rew, dtype=torch.float32), dones=torch.tensor(rng.random((T + 1, c.B)) < 0.05, dtype=torch.float32),
                filled=torch.tensor(rng.random((T, c.B)) < 0.9, dtype=torch.float32))


def seeded_state(c: Case):
    """the case's initial agents' networks and mixer: the oracle, the reference (fixture generation) and the device all start from these"""
    n_nets = 1 if c.sharing else c.N
    theta = seeded_params(lr, n_nets, c.D, A, c.seed)
    torch.manual_seed(c.seed)
    mix = qo.init_mixer_flat(c.N, c.N * c.D, 64, 32, c.hl)
    return qo.QmixOptState(theta.clone(), theta.clone(), mix.clone(), mix.clone(), [0] * c.N if c.sharing else list(range(c.N)), c.D, A,
                           hypernet_layers=c.hl, ret_ms=lr.RunningMeanStdRef((1,)) if c.standardise else None)


def hp_of(c: Case):
    return lr.DqnHP(target_update_interval_or_tau=c.tu)


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_reference(name):
    """three updates of the reference's QMixNetwork with each option from the same weights and batches: the loss of every update, all four
    parameter sets and the running return statistics"""
    g, c = reference_outputs("qmix_options_reference"), CASES[name]
    st = seeded_state(c)
    assert st.mix.numel() == qo.mixer_size(c.N, c.N * c.D, 64, 32, c.hl)
    rng = np.random.default_rng(c.seed)
    for u in range(3):
        got = qo.qmix_update(st, batch(rng, c), hp_of(c))
        want = float(g[f"{name}_loss"][u])
        assert abs(got["loss"] - want) <= 1e-5 * max(1.0, abs(want)), f"loss of update {u}"
    for mine, key in ((st.theta, "theta"), (st.theta_tgt, "theta_tgt"), (st.mix, "mix"), (st.mix_tgt, "mix_tgt")):
        assert np.quantile(np.abs(mine.numpy()[::STRIDE] - g[f"{name}_{key}"]), 0.999) < 1e-5, key
    if c.standardise:
        assert st.ret_ms.mean.shape == (c.B,)
        np.testing.assert_allclose(st.ret_ms.mean.numpy(), g[f"{name}_ret_mean"], rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(st.ret_ms.var.numpy(), g[f"{name}_ret_var"], rtol=1e-5, atol=1e-6)
        assert st.ret_ms.count == pytest.approx(float(g[f"{name}_ret_count"]), rel=1e-12)


def make_reference_outputs(ref, ref_shim):
    """tests/golden/qmix_options_reference.npz: the reference's QMixNetwork run on CASES (3 updates each)."""
    out = {}
    for name, c in CASES.items():
        st = seeded_state(c)
        kind, n_nets = ("networks", 1) if c.sharing else ("independent", c.N)
        spaces = ([ref_shim.Space(shape=(c.D,))] * c.N, [ref_shim.Space(n=A)] * c.N)
        cfg = ref_shim.dqn_cfg(target_update_interval_or_tau=c.tu, standardise_returns=c.standardise)
        model = ref.dqn_model.QMixNetwork(*spaces, cfg, [128, 128], c.sharing, False, True, dict(embed_dim=64, hypernet_layers=c.hl, hypernet_embed=32), "cpu")
        load_params(model, lr, (f"critic.{kind}", f"target.{kind}"), st.theta, n_nets, c.D, A)
        msd = {}
        for prefix in ("mixer", "target_mixer"):
            msd.update(qo.mixer_state_dict_from_flat(st.mix, prefix, c.N, c.N * c.D, 64, 32, c.hl))
        assert set(msd) <= set(model.state_dict()), sorted(set(msd) - set(model.state_dict()))[:4]
        model.load_state_dict(msd, strict=False)
        rng = np.random.default_rng(c.seed)
        losses = []
        for _ in range(3):
            b = batch(rng, c)
            losses.append(model.update(ref.dqn_train.Batch(b["obss"], b["actions"], b["rewards"], b["dones"], b["filled"], None))["loss"])
        sd = model.state_dict()
        out[f"{name}_loss"] = np.array(losses, np.float64)
        out[f"{name}_theta"] = lr.flat_from_state_dict(sd, f"critic.{kind}", n_nets).numpy()[::STRIDE]
        out[f"{name}_theta_tgt"] = lr.flat_from_state_dict(sd, f"target.{kind}", n_nets).numpy()[::STRIDE]
        out[f"{name}_mix"] = qo.mixer_flat_from_state_dict(sd, "mixer", c.hl).numpy()[::STRIDE]
        out[f"{name}_mix_tgt"] = qo.mixer_flat_from_state_dict(sd, "target_mixer", c.hl).numpy()[::STRIDE]
        if c.standardise:
            out[f"{name}_ret_mean"] = model.ret_ms.mean.numpy().copy()
            out[f"{name}_ret_var"] = model.ret_ms.var.numpy().copy()
            out[f"{name}_ret_count"] = np.float64(model.ret_ms.count)
    np.savez_compressed(os.path.join(GOLDEN_DIR, "qmix_options_reference.npz"), **out)


def coverage(n, s, e, hl, he=32):
    """marl_debug_qmix_coverage_layers: (parameter count, per-parameter write counts of the single-read and the tile decomposition)"""
    from codebase_b200 import _native as nat

    lib = nat.lib()
    npar = C.c_int64()
    nat.check(lib.marl_debug_qmix_coverage_layers(C.c_int32(n), C.c_int32(s), C.c_int32(e), C.c_int32(hl), C.c_int32(he), None, C.c_int64(0), C.byref(npar)),
              "marl_debug_qmix_coverage_layers")
    counts = (C.c_int32 * (2 * npar.value))()
    nat.check(lib.marl_debug_qmix_coverage_layers(C.c_int32(n), C.c_int32(s), C.c_int32(e), C.c_int32(hl), C.c_int32(he), counts, C.c_int64(2 * npar.value),
                                                  C.byref(npar)), "marl_debug_qmix_coverage_layers")
    c = np.ctypeslib.as_array(counts)
    return npar.value, c[: npar.value], c[npar.value:]


@pytest.mark.parametrize("n,s,e,he", [(2, 30, 64, 32), (2, 18, 64, 32), (4, 108, 64, 32), (3, 27, 32, 16), (8, 120, 64, 64), (2, 5, 4, 4), (5, 33, 36, 12)])
def test_one_layer_weight_gradient_decompositions_cover_every_parameter_exactly_once(n, s, e, he):
    """csrc/qmix.cuh's five-layer table: the micro-tiles of the single-read weight-gradient kernel and the 32 x 32 tiles each write every parameter
    of the one-layer mixer exactly once, and the parameter count is the reference's (hypernet_embed does not matter)"""
    npar, single, tiles = coverage(n, s, e, 1, he)
    assert npar == qo.mixer_size(n, s, e, he, 1) == n * e * s + n * e + 3 * (e * s + e) + e + 1
    assert (single == 1).all(), "single-read form"
    assert (tiles == 1).all(), "tile form"


def test_two_layer_coverage_through_the_new_entry_point_is_the_old_one():
    from codebase_b200 import _native as nat

    lib = nat.lib()
    old = C.c_int64()
    nat.check(lib.marl_debug_qmix_coverage(C.c_int32(4), C.c_int32(108), C.c_int32(64), C.c_int32(32), None, C.c_int64(0), C.byref(old)), "marl_debug_qmix_coverage")
    npar, single, tiles = coverage(4, 108, 64, 2)
    assert npar == old.value == qo.mixer_size(4, 108, 64, 32)
    assert (single == 1).all() and (tiles == 1).all()


def test_other_hypernetwork_depths_are_refused():
    from codebase_b200 import _native as nat

    lib = nat.lib()
    npar = C.c_int64()
    for hl in (0, 3):
        rc = lib.marl_debug_qmix_coverage_layers(C.c_int32(2), C.c_int32(18), C.c_int32(64), C.c_int32(hl), C.c_int32(32), None, C.c_int64(0), C.byref(npar))
        assert rc != 0 and b"hypernet_layers" in lib.marl_last_error()
    with pytest.raises(ValueError, match="hypernet_layers"):
        qo.mixer_shapes(2, 18, 64, 32, 3)


def test_host_class_checks_the_mixer_configuration_before_any_native_call():
    """every configuration the kernels implement passes codebase_b200.dqn.model.check_mixing (both forms, both standardise_returns values, the
    4-agent env); other depths and out-of-range widths raise NotImplementedError naming the configuration"""
    from codebase_b200.dqn import model as M

    obs = lambda n, d: [types.SimpleNamespace(shape=(d,), n=None)] * n
    for hl in (1, 2):
        for std in (False, True):
            M.check_mixing(obs(4, 27), dict(embed_dim=64, hypernet_layers=hl, hypernet_embed=32), std)
            M.check_mixing(obs(2, 15), dict(embed_dim=36, hypernet_layers=hl, hypernet_embed=32), std)
    M.check_mixing(obs(8, 32), dict(embed_dim=64, hypernet_layers=1, hypernet_embed=0), False)   # hypernet_embed is ignored with one layer
    for mixing, n, d, why in ((dict(embed_dim=64, hypernet_layers=3, hypernet_embed=32), 2, 15, "hypernet_layers must be 1 or 2"),
                              (dict(embed_dim=64, hypernet_layers=2, hypernet_embed=0), 2, 15, "hypernet_embed"),
                              (dict(embed_dim=66, hypernet_layers=1, hypernet_embed=32), 2, 15, "embed_dim"),
                              (dict(embed_dim=64, hypernet_layers=1, hypernet_embed=32), 9, 15, "n_agents"),
                              (dict(embed_dim=64, hypernet_layers=1, hypernet_embed=32), 4, 65, "state_dim")):
        with pytest.raises(NotImplementedError, match=why):
            M.check_mixing(obs(n, d), mixing, True)


def test_one_layer_host_layout_and_keys():
    """codebase_b200.dqn.model builds the one-layer mixer's Linear layers in the reference's order and names them with its keys"""
    from codebase_b200.dqn import model as M

    assert M.mixer_shapes(4, 108, 64, 32, 1) == qo.mixer_shapes(4, 108, 64, 32, 1) == ((256, 108), (64, 108), (64, 108), (64, 108), (1, 64))
    assert M.mixer_keys(1) == qo.mixer_keys(1) == ("hyper_w_1", "hyper_w_final", "hyper_b_1", "V.0", "V.2")
    assert M.mixer_shapes(2, 30, 64, 32) == qo.mixer_shapes(2, 30, 64, 32) == qr.mixer_shapes(2, 30, 64, 32) and M.mixer_keys() == qr.MIXER_KEYS
    torch.manual_seed(5)
    flat = qo.init_mixer_flat(2, 18, 64, 32, 1)
    torch.manual_seed(5)
    w1, w_final = torch.nn.Linear(18, 128), torch.nn.Linear(18, 64)
    assert torch.equal(flat[: 128 * 18], w1.weight.data.reshape(-1)) and torch.equal(flat[128 * 19: 128 * 19 + 64 * 18], w_final.weight.data.reshape(-1))


if __name__ == "__main__":   # MARL_REFERENCE_ROOT=<checkout> python -m tests.test_qmix_options
    from oracle import ref_shim

    make_reference_outputs(ref_shim.load(), ref_shim)

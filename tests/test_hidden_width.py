"""Hidden widths other than 128 (`layers: [H, H]`, 1 <= H <= 128) in all seven learners, CPU side: the oracle (oracle/learner_ref.py and
oracle/qmix_ref.py run with the width-H networks of tests/hidden_width_ref.py) against what the reference's own QNetwork / VDNetwork / QMixNetwork / A2CNetwork /
PPONetwork computed at those widths (tests/golden/hidden_width_reference.npz), the host-side width check, and the state_dict names and shapes.
The CUDA path is checked in tests/test_hidden_width_gpu.py.

`MARL_REFERENCE_ROOT=<reference checkout> python -m tests.test_hidden_width` regenerates the fixture."""
import os
import re
import types
from collections import namedtuple

import numpy as np
import pytest
import torch

from oracle import learner_ref as lr
from oracle import qmix_ref as qr
from tests import hidden_width_ref as hr
from tests.helpers import GOLDEN, STRIDE, ac_batch, ac_oracle_batch, random_store, reference_outputs, space

N, A = 2, 6
DQN_T, DQN_D, DQN_B, DQN_CAP = 6, 9, 8, 12
AC_T, AC_D, AC_P = 10, 9, 6
MIXING = dict(embed_dim=64, hypernet_layers=2, hypernet_embed=32)
UPDATES = 2
EPOCHS = 2

# DQN family: (mixer 0 IDQN / 1 VDN / 2 QMIX, recurrent, hidden, parameter sharing, target_update_interval_or_tau, seed)
DQN_CASES = {
    "idqn_64": (0, False, 64, False, 200, 41),
    "vdn_64": (1, False, 64, True, 0.05, 42),
    "qmix_64": (2, False, 64, False, 200, 43),
    "idqn_gru_64": (0, True, 64, False, 200, 44),
}
# actor-critic: (class, actor hidden, actor recurrent, critic hidden, critic recurrent, centralised critic, sharing, grad_clip, seed)
AC_CASES = {
    "ia2c_64_37": ("A2CNetwork", 64, False, 37, False, False, False, 0.0, 51),
    "mappo_gru64_central32": ("PPONetwork", 64, True, 32, False, True, True, 0.5, 52),
}
AC_STEPS = (0, 2)


# ---- the cases --------------------------------------------------------------------------------------------------------------------------------
def dqn_setup(name):
    """(oracle state, hp, replay store in the device layout, per-update episode indices)"""
    mixer, rnn, H, sharing, tu, seed = DQN_CASES[name]
    n_nets = 1 if sharing else N
    agent_net = [0] * N if sharing else list(range(N))
    torch.manual_seed(seed)
    theta = hr.init_gru(n_nets, DQN_D, A, H) if rnn else hr.init_mlp(n_nets, DQN_D, A, H, generator=torch.Generator().manual_seed(seed))
    rng = np.random.default_rng(seed)
    store = random_store(rng, DQN_CAP, N, DQN_T, DQN_D, coop=mixer != 0, A=A)
    idx = rng.integers(0, DQN_CAP, size=(UPDATES, DQN_B)).astype(np.int32)
    if mixer == 2:
        mix = qr.init_mixer_flat(N, N * DQN_D, MIXING["embed_dim"], MIXING["hypernet_embed"])
        st = qr.QmixState(theta.clone(), theta.clone(), mix.clone(), mix.clone(), agent_net, DQN_D, A, MIXING["embed_dim"], MIXING["hypernet_embed"])
    else:
        st = lr.DqnState(theta.clone(), theta.clone(), agent_net, DQN_D, A)
    return st, lr.DqnHP(target_update_interval_or_tau=tu, mixer=mixer), store, idx


def dqn_oracle_update(name, st, batch, hp):
    mixer, rnn = DQN_CASES[name][:2]
    with hr.networks([(DQN_D, A)] if rnn else []):
        return qr.qmix_update(st, batch, hp) if mixer == 2 else lr.dqn_update(st, batch, hp)


def ac_networks(name):
    """learner_ref's A2C / PPO functions with each part's network kind: the actor (AC_D -> A) and the critic (its input width -> 1) are told
    apart by their widths; the hidden width of each call is read from its flat vector (hidden_width_ref.width_of)"""
    _, _, arnn, _, crnn, central, _, _, _ = AC_CASES[name]
    return hr.networks([(AC_D, A)] * arnn + [(N * AC_D if central else AC_D, 1)] * crnn)


def ac_setup(name):
    """(oracle state, hp, batches in the device layout)"""
    _, ah, arnn, ch, crnn, central, sharing, clip, seed = AC_CASES[name]
    n_nets = 1 if sharing else N
    nets = [0] * N if sharing else list(range(N))
    CD = N * AC_D if central else AC_D
    torch.manual_seed(seed)
    actor = hr.init_gru(n_nets, AC_D, A, ah) if arnn else hr.init_mlp(n_nets, AC_D, A, ah)
    critic = hr.init_gru(n_nets, CD, 1, ch) if crnn else hr.init_mlp(n_nets, CD, 1, ch)
    st = lr.A2CState(actor, critic.clone(), critic.clone(), nets, nets, AC_D, A, centralised=central)
    hp = lr.A2CHP(grad_clip=clip, target_update_interval_or_tau=2)
    rng = np.random.default_rng(seed)
    return st, hp, [ac_batch(rng, AC_P, N, AC_T, AC_D, A) for _ in AC_STEPS]


def ac_oracle_update(name, st, batch, hp, step):
    with ac_networks(name):
        if AC_CASES[name][0] == "PPONetwork":
            return lr.ppo_update(st, batch, hp, step, EPOCHS, 0.2)
        return lr.a2c_update(st, batch, hp, step)


# ---- the oracle against the reference ---------------------------------------------------------------------------------------------------------
def _quantile_close(mine, want, what):
    d = np.abs(np.asarray(mine, np.float64)[::STRIDE] - np.asarray(want, np.float64))
    assert np.quantile(d, 0.999) < 1e-5, (what, float(d.max()))


@pytest.mark.parametrize("name", list(DQN_CASES))
def test_oracle_matches_reference_dqn(name):
    g = reference_outputs("hidden_width_reference")
    st, hp, store, idx = dqn_setup(name)
    for u in range(UPDATES):
        got = dqn_oracle_update(name, st, lr.batch_from_store(store, idx[u]), hp)
        want = float(g[f"{name}_loss"][u])
        assert abs(got["loss"] - want) <= 1e-5 * max(1.0, abs(want)), (u, got["loss"], want)
    _quantile_close(st.theta.numpy(), g[f"{name}_theta"], "theta")
    _quantile_close(st.theta_tgt.numpy(), g[f"{name}_theta_tgt"], "theta_tgt")
    if DQN_CASES[name][0] == 2:
        _quantile_close(st.mix.numpy(), g[f"{name}_mix"], "mix")


@pytest.mark.parametrize("name", list(AC_CASES))
def test_oracle_matches_reference_ac(name):
    g = reference_outputs("hidden_width_reference")
    st, hp, batches = ac_setup(name)
    metrics = []
    for step, s in zip(AC_STEPS, batches):
        got = ac_oracle_update(name, st, ac_oracle_batch(s), hp, step)
        metrics.append([got[k] for k in ("loss", "actor_loss", "value_loss", "entropy")])
    assert np.allclose(metrics, g[f"{name}_metrics"], rtol=1e-5, atol=1e-5), (metrics, g[f"{name}_metrics"])
    for mine, key in ((st.actor, "actor"), (st.critic, "critic"), (st.target, "target")):
        _quantile_close(mine.numpy(), g[f"{name}_{key}"], key)


def test_width_h_networks_at_128_are_the_oracles():
    """at H = 128 the width-H restatement is the 128-wide oracle's network: same sizes, same initial weights, same outputs; widths are read
    back from a flat vector's length"""
    from oracle import gru_ref as gr

    assert hr.net_size(15, 6, 128) == lr.net_size(15, 6) and hr.net_size(15, 6, 128, True) == gr.net_size(15, 6) == 101_894
    for H in (1, 37, 64, 100, 128):
        for rnn in (False, True):
            assert hr.width_of(torch.zeros(2 * hr.net_size(15, 6, H, rnn)), [0, 1], 15, 6, rnn) == H
    assert hr.width_of(torch.zeros(2 * hr.net_size(15, 6, 64) + 1), [0, 1], 15, 6) is None
    g = torch.Generator
    assert torch.equal(hr.init_mlp(2, 15, 6, 128, generator=g().manual_seed(3)), lr.init_flat(2, 15, 6, generator=g().manual_seed(3)))
    torch.manual_seed(4); a = hr.init_gru(1, 15, 6, 128)
    torch.manual_seed(4); b = gr.init_flat(1, 15, 6)
    assert torch.equal(a, b)
    x = torch.randn(5, 3, 15)
    assert torch.equal(hr.agents_forward(b, [0], [x], 15, 6, True)[0], gr.agents_forward(b, [0], [x], 15, 6)[0])
    flat = lr.init_flat(2, 15, 6)
    assert torch.equal(hr.agents_forward(flat, [0, 1], [x, x], 15, 6)[1], lr.agents_forward(flat, [0, 1], [x, x], 15, 6)[1])


# ---- the host-side check ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layers", [[1, 1], [37, 37], [64, 64], [128, 128]])
def test_host_check_accepts(layers):
    from codebase_b200 import learner as L

    assert L.hidden_width(layers) == layers[0]
    assert L.hidden_width(layers, "actor.layers", use_rnn=True) == layers[0]


@pytest.mark.parametrize("layers", [[129, 129], [64, 32], [64], [64, 64, 64], [0, 0], []])
def test_host_check_refuses(layers):
    from codebase_b200 import learner as L

    with pytest.raises(NotImplementedError, match=re.escape(f"layers={layers}") + r".*1 <= H <= 128"):
        L.hidden_width(layers)


def _dqn_cfg():
    return types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=1.0, double_q=True, target_update_interval_or_tau=200,
                                 standardise_returns=False)


def _net(layers, use_rnn=False, centralised=False):
    return types.SimpleNamespace(layers=layers, parameter_sharing=False, use_rnn=use_rnn, use_orthogonal_init=True, centralised=centralised)


@pytest.mark.parametrize("layers", [[129, 129], [64, 32], [64], [64, 64, 64]])
def test_constructors_refuse_before_any_native_call(layers, monkeypatch):
    """the width check runs first in every learner's constructor: no device and no library are needed to be refused"""
    from codebase_b200 import _native as nat
    from codebase_b200.ac import model as AM
    from codebase_b200.dqn import model as M

    def no_lib():
        raise AssertionError("the native library was reached")

    monkeypatch.setattr(nat, "lib", no_lib)
    obs, act = [space(shape=(9,))] * 2, [space(n=6)] * 2
    for cls in (M.QNetwork, M.VDNetwork):
        for rnn in (False, True):
            with pytest.raises(NotImplementedError, match=r"layers="):
                cls(obs, act, _dqn_cfg(), layers, False, rnn, True, "cuda")
    with pytest.raises(NotImplementedError, match=r"layers="):
        M.QMixNetwork(obs, act, _dqn_cfg(), layers, False, False, True, MIXING, "cuda")
    ac_cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=0.0, n_steps=5, entropy_coef=0.001, value_loss_coef=0.5,
                                   target_update_interval_or_tau=200, standardise_returns=False, num_epochs=4, ppo_clip=0.2)
    for cls in (AM.A2CNetwork, AM.PPONetwork):
        with pytest.raises(NotImplementedError, match=r"actor\.layers="):
            cls(obs, act, ac_cfg, _net(layers), _net([64, 64]), "cuda")
        with pytest.raises(NotImplementedError, match=r"critic\.layers="):
            cls(obs, act, ac_cfg, _net([64, 64]), _net(layers, use_rnn=True, centralised=True), "cuda")


# ---- state_dict names and shapes --------------------------------------------------------------------------------------------------------------
def test_layout_tables_match_the_reference_state_dict_at_64():
    """the reference's FCNetwork / RNNNetwork at layers [64, 64]: the names and shapes the flat layout converts to (recorded in the fixture)"""
    from codebase_b200 import learner as L

    g = reference_outputs("hidden_width_reference")
    mlp = L.flat_to_state_dict(torch.zeros(2 * hr.net_size(DQN_D, A, 64)), "critic.independent", 2, L.mlp_shapes(DQN_D, A, 64))
    rnn = L.flat_to_state_dict(torch.zeros(2 * hr.net_size(DQN_D, A, 64, True)), "critic.independent", 2, L.rnn_shapes(DQN_D, A, 64))
    for sd, key in ((mlp, "idqn_64"), (rnn, "idqn_gru_64")):
        names = [str(x) for x in g[f"{key}_sd_names"]]
        shapes = [tuple(int(v) for v in s if v >= 0) for s in g[f"{key}_sd_shapes"]]
        mine = [(k, tuple(v.shape)) for k, v in sd.items() if k.startswith("critic.")]
        assert mine == list(zip(names, shapes))
    flat = torch.randn(2 * hr.net_size(DQN_D, A, 64, True))
    shapes = L.rnn_shapes(DQN_D, A, 64)
    assert torch.equal(L.state_dict_to_flat(L.flat_to_state_dict(flat, "c", 2, shapes), "c", 2, shapes), flat)
    flat = torch.randn(2 * hr.net_size(DQN_D, A, 37))
    shapes = L.mlp_shapes(DQN_D, A, 37)
    assert torch.equal(L.state_dict_to_flat(L.flat_to_state_dict(flat, "c", 2, shapes), "c", 2, shapes), flat)


def test_host_initialisation_at_37():
    """init_flat_params / init_flat_rnn_params build the compact layout of width H (P = H*in + H + H*H + H + out*H + out)"""
    from codebase_b200 import learner as L

    assert L.init_flat_params(2, DQN_D, A, True, 37).numel() == 2 * hr.net_size(DQN_D, A, 37)
    assert L.init_flat_rnn_params(1, DQN_D, A, True, 37).numel() == hr.net_size(DQN_D, A, 37, True)
    w3 = hr.split_net(L.init_flat_params(1, DQN_D, A, True, 37), DQN_D, A, 37)[4]
    assert torch.allclose(w3 @ w3.T, 2.0 * torch.eye(A), atol=1e-5)


def test_yaml_defaults_stay_128():
    from codebase_b200.config import compose

    for alg in ("idqn", "vdn", "qmix"):
        c = compose([f"+algorithm={alg}", "env.name=lbforaging:Foraging-8x8-2p-3f-v3", "env.time_limit=25"])
        assert list(c.algorithm.model.layers) == [128, 128]
    c = compose(["+algorithm=idqn", "env.name=lbforaging:Foraging-8x8-2p-3f-v3", "env.time_limit=25", "algorithm.model.layers=[64,64]"])
    assert list(c.algorithm.model.layers) == [64, 64]
    for alg in ("ia2c", "ippo", "maa2c", "mappo"):
        c = compose([f"+algorithm={alg}", "env.name=lbforaging:Foraging-8x8-2p-3f-v3", "env.time_limit=25"])
        assert list(c.algorithm.model.actor.layers) == [128, 128] and list(c.algorithm.model.critic.layers) == [128, 128]


# ---- fixture generation -----------------------------------------------------------------------------------------------------------------------
def make_reference_outputs(ref, ref_shim):
    """tests/golden/hidden_width_reference.npz: the reference's learners at the cases' widths, loaded with the cases' initial weights"""
    out = {}
    ACBatch = namedtuple("Batch", ["obss", "actions", "rewards", "dones", "filled", "action_masks"])
    for name, (mixer, rnn, H, sharing, tu, seed) in DQN_CASES.items():
        st, hp, store, idx = dqn_setup(name)
        cfg = ref_shim.dqn_cfg(target_update_interval_or_tau=tu)
        spaces = ([ref_shim.Space(shape=(DQN_D,))] * N, [ref_shim.Space(n=A)] * N)
        if mixer == 2:
            model = ref.dqn_model.QMixNetwork(*spaces, cfg, [H, H], sharing, rnn, True, MIXING, "cpu")
        else:
            model = (ref.dqn_model.VDNetwork if mixer == 1 else ref.dqn_model.QNetwork)(*spaces, cfg, [H, H], sharing, rnn, True, "cpu")
        kind, n_nets = ("networks", 1) if sharing else ("independent", N)
        sd = {**hr.state_dict_from_flat(st.theta, f"critic.{kind}", n_nets, DQN_D, A, H, rnn),
              **hr.state_dict_from_flat(st.theta, f"target.{kind}", n_nets, DQN_D, A, H, rnn)}
        if mixer == 2:
            for prefix in ("mixer", "target_mixer"):
                sd.update(qr.mixer_state_dict_from_flat(st.mix, prefix, N, N * DQN_D, MIXING["embed_dim"], MIXING["hypernet_embed"]))
        ref_sd = model.state_dict()
        assert set(sd) <= set(ref_sd) and all(tuple(ref_sd[k].shape) == tuple(v.shape) for k, v in sd.items()), name
        model.load_state_dict(sd, strict=False)
        if name in ("idqn_64", "idqn_gru_64"):   # the reference's own names and shapes of the agents' networks
            names = [k for k in ref_sd if k.startswith("critic.")]
            out[f"{name}_sd_names"] = np.array(names)
            out[f"{name}_sd_shapes"] = np.array([list(ref_sd[k].shape) + [-1] * (2 - ref_sd[k].dim()) for k in names], np.int64)
        losses = []
        for u in range(UPDATES):
            b = lr.batch_from_store(store, idx[u])
            losses.append(float(model.update(ref.dqn_train.Batch(b["obss"], b["actions"], b["rewards"], b["dones"], b["filled"], None))["loss"]))
        out[f"{name}_loss"] = np.array(losses, np.float64)
        sd = model.state_dict()
        out[f"{name}_theta"] = hr.flat_from_state_dict(sd, f"critic.{kind}", n_nets, rnn).numpy()[::STRIDE]
        out[f"{name}_theta_tgt"] = hr.flat_from_state_dict(sd, f"target.{kind}", n_nets, rnn).numpy()[::STRIDE]
        if mixer == 2:
            out[f"{name}_mix"] = qr.mixer_flat_from_state_dict(sd, "mixer").numpy()[::STRIDE]
    for name, (cls, ah, arnn, ch, crnn, central, sharing, clip, seed) in AC_CASES.items():
        st, hp, batches = ac_setup(name)
        cfg = ref_shim.a2c_cfg(grad_clip=clip or False, num_epochs=EPOCHS, ppo_clip=0.2, target_update_interval_or_tau=2)
        anet = types.SimpleNamespace(layers=[ah, ah], parameter_sharing=sharing, use_rnn=arnn, use_orthogonal_init=True, centralised=False)
        cnet = types.SimpleNamespace(layers=[ch, ch], parameter_sharing=sharing, use_rnn=crnn, use_orthogonal_init=True, centralised=central)
        model = getattr(ref.ac_model, cls)([ref_shim.Space(shape=(AC_D,))] * N, [ref_shim.Space(n=A)] * N, cfg, anet, cnet, "cpu")
        kind, n_nets = ("networks", 1) if sharing else ("independent", N)
        CD = N * AC_D if central else AC_D
        sd = {**hr.state_dict_from_flat(st.actor, f"actor.{kind}", n_nets, AC_D, A, ah, arnn),
              **hr.state_dict_from_flat(st.critic, f"critic.{kind}", n_nets, CD, 1, ch, crnn),
              **hr.state_dict_from_flat(st.critic, f"target_critic.{kind}", n_nets, CD, 1, ch, crnn)}
        assert set(sd) == set(model.state_dict()), sorted(set(sd) ^ set(model.state_dict()))[:4]
        model.load_state_dict(sd)
        metrics = []
        for step, s in zip(AC_STEPS, batches):
            b = ac_oracle_batch(s)
            res = model.update(ACBatch(b["obss"], b["actions"], b["rewards"], b["dones"].bool(), b["filled"], None), step)
            metrics.append([float(res[k]) for k in ("loss", "actor_loss", "value_loss", "entropy")])
        out[f"{name}_metrics"] = np.array(metrics, np.float64)
        sd = model.state_dict()
        out[f"{name}_actor"] = hr.flat_from_state_dict(sd, f"actor.{kind}", n_nets, arnn).numpy()[::STRIDE]
        out[f"{name}_critic"] = hr.flat_from_state_dict(sd, f"critic.{kind}", n_nets, crnn).numpy()[::STRIDE]
        out[f"{name}_target"] = hr.flat_from_state_dict(sd, f"target_critic.{kind}", n_nets, crnn).numpy()[::STRIDE]
    np.savez_compressed(os.path.join(GOLDEN, "hidden_width_reference.npz"), **out)


if __name__ == "__main__":
    from oracle import ref_shim

    torch.set_num_threads(1)
    make_reference_outputs(ref_shim.load(), ref_shim)

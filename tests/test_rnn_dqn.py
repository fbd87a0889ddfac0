"""Recurrent (GRU) agent networks of IDQN / VDN / QMIX (algorithm.model.use_rnn=True), CPU side: the oracle restatement (oracle/gru_ref.py)
against outputs of the reference project's own QNetwork / VDNetwork / QMixNetwork stored under tests/golden/rnn_*.npz, the host-side parameter
layout and initialisation rule, config composition and the exported symbols.  The device kernels are checked in test_rnn_dqn_gpu.py."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import gru_ref as gr
from oracle import learner_ref as lr
from oracle import qmix_ref as qr
from tests.helpers import STRIDE, random_store

N, T, D, A, B, CAP = 2, 6, 9, 6, 8, 12
GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MIXING = dict(embed_dim=64, hypernet_layers=2, hypernet_embed=32)

# name: (mixer, parameter sharing, hyper-parameters, standardise_returns, seed)
CASES = {
    "idqn_indep": (0, False, dict(double_q=True, target_update_interval_or_tau=2.0, grad_clip=1.0), False, 101),
    "idqn_shared": (0, True, dict(double_q=False, target_update_interval_or_tau=0.05, grad_clip=0.0), False, 102),
    "vdn_indep": (1, False, dict(double_q=True, target_update_interval_or_tau=2.0, grad_clip=1.0), False, 103),
    "qmix_shared": (2, True, dict(double_q=True, target_update_interval_or_tau=2.0, grad_clip=1.0), False, 104),
    "idqn_standardise": (0, False, dict(double_q=True, target_update_interval_or_tau=0.05, grad_clip=1.0), True, 105),
}


def golden_path(name):
    return os.path.join(GOLDEN_DIR, f"rnn_{name}.npz")


def case_setup(name):
    """(hp, agent_net, n_nets, theta0, mix0 or None, store, idx[3][B], act-step observations) of a case; parameters regenerated from the seed"""
    mixer, sharing, kw, standardise, seed = CASES[name]
    hp = lr.DqnHP(lr=3e-4, gamma=0.99, mixer=min(mixer, 1), **kw)
    n_nets = 1 if sharing else N
    torch.manual_seed(seed)
    theta0 = gr.init_flat(n_nets, D, A)
    mix0 = qr.init_mixer_flat(N, N * D, MIXING["embed_dim"], MIXING["hypernet_embed"]) if mixer == 2 else None
    rng = np.random.default_rng(seed)
    store = random_store(rng, CAP, N, T, D, coop=mixer > 0, A=A)
    store["obs"] = (store["obs"] / 6.0).astype(np.float32)   # LBF-like magnitudes keep the GRU away from saturation
    idx = rng.integers(0, CAP, size=(3, B)).astype(np.int32)
    act_obs = (rng.integers(-1, 12, size=(10, N, D)) / 6.0).astype(np.float32)
    return hp, ([0] * N if sharing else list(range(N))), n_nets, theta0, mix0, store, idx, act_obs


def oracle_state(name, theta0, mix0, agent_net):
    mixer, _, _, standardise, _ = CASES[name]
    if mixer == 2:
        return qr.QmixState(theta0.clone(), theta0.clone(), mix0.clone(), mix0.clone(), agent_net, D, A, **{k: MIXING[k] for k in ("embed_dim", "hypernet_embed")})
    st = lr.DqnState(theta0.clone(), theta0.clone(), agent_net, D, A)
    if standardise:
        st.ret_ms = lr.RunningMeanStdRef((N,))
    return st


def oracle_update(name, st, batch, hp):
    return gr.qmix_update(st, batch, hp) if CASES[name][0] == 2 else gr.dqn_update(st, batch, hp)


def make_golden():
    """Regenerates tests/golden/rnn_*.npz from the reference project (MARL_REFERENCE_ROOT): its QNetwork / VDNetwork / QMixNetwork with
    use_rnn=True, loaded with each case's parameters, run through three updates and ten act() steps."""
    from oracle import ref_shim

    ref = ref_shim.load()
    for name, (mixer, sharing, kw, standardise, seed) in CASES.items():
        hp, agent_net, n_nets, theta0, mix0, store, idx, act_obs = case_setup(name)
        cfg = ref_shim.dqn_cfg(standardise_returns=standardise, **kw)
        spaces = ([ref_shim.Space(shape=(D,))] * N, [ref_shim.Space(n=A)] * N)
        if mixer == 2:
            model = ref.dqn_model.QMixNetwork(*spaces, cfg, [128, 128], sharing, True, True, MIXING, "cpu")
        else:
            cls = ref.dqn_model.VDNetwork if mixer == 1 else ref.dqn_model.QNetwork
            model = cls(*spaces, cfg, [128, 128], sharing, True, True, "cpu")
        kind = "networks" if sharing else "independent"
        sd = {**gr.state_dict_from_flat(theta0, f"critic.{kind}", n_nets, D, A), **gr.state_dict_from_flat(theta0, f"target.{kind}", n_nets, D, A)}
        if mixer == 2:
            sd.update(qr.mixer_state_dict_from_flat(mix0, "mixer", N, N * D, 64, 32)); sd.update(qr.mixer_state_dict_from_flat(mix0, "target_mixer", N, N * D, 64, 32))
        missing = set(sd) - set(model.state_dict())
        assert not missing, sorted(missing)[:4]
        model.load_state_dict(sd, strict=False)
        critic = list(model.critic.parameters())
        out = dict(stride=np.int32(STRIDE), theta0=theta0.numpy()[::STRIDE], idx=idx, **{f"store_{k}": v for k, v in store.items()})
        # ten consecutive act() steps of one env from init_hiddens, at the initial parameters: the network pass act() runs (dqn/model.py:96-99) and the hiddens it returns
        hid = model.init_hiddens(1)
        qs, hs = [], []
        for s in range(10):
            with torch.no_grad():
                values, _ = model.critic([torch.tensor(act_obs[s, a]).view(1, 1, -1) for a in range(N)], hid)
            _, hid = model.act([act_obs[s, a] for a in range(N)], hid, 0.0)
            qs.append(np.stack([v.reshape(-1).numpy() for v in values])); hs.append(np.stack([h.reshape(-1).numpy() for h in hid]))
        out.update(act_obs=act_obs, act_q=np.stack(qs), act_h=np.stack(hs))
        losses = []
        for u in range(3):
            b = lr.batch_from_store(store, idx[u])
            losses.append(model.update(ref.dqn_train.Batch(b["obss"], b["actions"], b["rewards"], b["dones"], b["filled"], None))["loss"])
            if u == 0:   # after clip_grad_norm_: the gradient Adam consumed
                out["grad1"] = torch.cat([p.grad.reshape(-1) for p in critic]).numpy()[::STRIDE]
        out["loss"] = np.array(losses, np.float64)
        sd = model.state_dict()
        out["theta3"] = gr.flat_from_state_dict(sd, f"critic.{kind}", n_nets).numpy()[::STRIDE]
        out["theta_tgt3"] = gr.flat_from_state_dict(sd, f"target.{kind}", n_nets).numpy()[::STRIDE]
        out["m3"] = torch.cat([model.optimizer.state[p]["exp_avg"].reshape(-1) for p in critic]).numpy()[::STRIDE]
        out["v3"] = torch.cat([model.optimizer.state[p]["exp_avg_sq"].reshape(-1) for p in critic]).numpy()[::STRIDE]
        if standardise:
            out.update(ret_mean=model.ret_ms.mean.numpy(), ret_var=model.ret_ms.var.numpy(), ret_count=np.float64(model.ret_ms.count))
        np.savez_compressed(golden_path(name), **out)


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_reference_golden(name):
    """three updates and ten act() steps of the reference's recurrent learner, recorded under tests/golden: losses, the first (clipped)
    gradient, Adam m / v, parameters, target, return statistics, act-step Q-values and hiddens -- all to 1e-5"""
    g = np.load(golden_path(name))
    hp, agent_net, n_nets, theta0, mix0, _, idx, _ = case_setup(name)
    assert np.array_equal(theta0.numpy()[::STRIDE], g["theta0"]), "the seeded initial parameters differ from the ones the fixture was made from"
    store = {k: g[f"store_{k}"] for k in ("obs", "act", "rew", "done", "filled")}
    st = oracle_state(name, theta0, mix0, agent_net)
    for u in range(3):
        res = oracle_update(name, st, lr.batch_from_store(store, g["idx"][u]), hp)
        assert abs(res["loss"] - float(g["loss"][u])) <= 1e-5 * max(1.0, abs(float(g["loss"][u]))), (u, res["loss"], float(g["loss"][u]))
        if u == 0:
            grad = res.get("grad_clipped")
            if grad is None:   # qmix_update returns the raw gradient: clip it as the reference's clip_grad_norm_ did
                coef, _ = lr.clip_coef(res["grad"], hp.grad_clip) if hp.grad_clip else (1.0, None)
                grad = res["grad"] * coef
            np.testing.assert_allclose(grad.numpy()[::STRIDE], g["grad1"], rtol=0, atol=1e-5 * max(1.0, float(np.abs(g["grad1"]).max())))
    for mine, key, tol in ((st.theta, "theta3", 1e-5), (st.theta_tgt, "theta_tgt3", 1e-5)):
        np.testing.assert_allclose(mine.numpy()[::STRIDE], g[key], rtol=0, atol=tol, err_msg=key)
    # Adam state relative to each tensor's scale.  v holds squared gradients: a relative gradient difference e (the restated GRU sums in another
    # order than nn.GRU: ~1e-5 on the largest elements) is 2e in v, and three steps add up
    for mine, key, tol in ((st.m, "m3", 2e-5), (st.v, "v3", 6e-5)):
        want = g[key]
        err, scale = float(np.abs(mine.numpy()[::STRIDE] - want).max()), max(float(np.abs(want).max()), 1e-30)
        assert err <= tol * scale, (key, err, scale)
    if CASES[name][3]:
        np.testing.assert_allclose(st.ret_ms.mean.numpy(), g["ret_mean"], rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(st.ret_ms.var.numpy(), g["ret_var"], rtol=1e-5)
        assert abs(st.ret_ms.count - float(g["ret_count"])) < 1e-9
    q, h = gr.act_steps(theta0, agent_net, torch.tensor(g["act_obs"]).unsqueeze(1), D, A)
    np.testing.assert_allclose(q[:, 0].numpy(), g["act_q"], rtol=0, atol=1e-5)
    np.testing.assert_allclose(h[:, 0].numpy(), g["act_h"], rtol=0, atol=1e-5)


def test_fixtures_stay_small():
    for name in CASES:
        assert os.path.getsize(golden_path(name)) < 1 << 20, name


def test_rnn_layout_table_round_trip_uses_reference_keys():
    from codebase_b200 import learner as L

    D_, A_ = 15, 6
    flat = torch.randn(2 * gr.net_size(D_, A_))
    assert gr.net_size(D_, A_) == 101_894
    sd = L.flat_to_state_dict(flat, "critic.independent", 2, L.rnn_shapes(D_, A_))
    assert list(sd)[:8] == [f"critic.independent.0.{n}" for n in gr.NAMES]
    shapes = {k.split(".", 3)[3]: tuple(v.shape) for k, v in sd.items() if k.startswith("critic.independent.1.")}
    assert shapes == {"first_layer.weight": (128, D_), "first_layer.bias": (128,), "rnn.weight_ih_l0": (384, 128), "rnn.weight_hh_l0": (384, 128),
                      "rnn.bias_ih_l0": (384,), "rnn.bias_hh_l0": (384,), "final_layer.weight": (A_, 128), "final_layer.bias": (A_,)}
    assert torch.equal(L.state_dict_to_flat(sd, "critic.independent", 2, L.rnn_shapes(D_, A_)), flat)
    assert torch.equal(gr.flat_from_state_dict(sd, "critic.independent", 2), flat)


def test_host_initialisation_rule():
    """use_orthogonal_init touches final_layer only (orthogonal, gain sqrt 2, zero bias); first_layer keeps nn.Linear's default, the GRU
    PyTorch's uniform(+-1/sqrt(128))"""
    from codebase_b200 import learner as L

    torch.manual_seed(3)
    D_, A_ = 15, 6
    parts = dict(zip(gr.NAMES, gr.split_net(L.init_flat_rnn_params(1, D_, A_, True), D_, A_)))
    w3 = parts["final_layer.weight"]
    assert torch.allclose(w3 @ w3.T, 2.0 * torch.eye(A_), atol=1e-5) and torch.all(parts["final_layer.bias"] == 0)
    bound = 1 / math.sqrt(128)
    for k in ("rnn.weight_ih_l0", "rnn.weight_hh_l0", "rnn.bias_ih_l0", "rnn.bias_hh_l0"):
        assert float(parts[k].abs().max()) <= bound and float(parts[k].abs().max()) > 0.9 * bound, k
    w1 = parts["first_layer.weight"]
    assert float(w1.abs().max()) <= 1 / math.sqrt(D_) and not torch.allclose(w1 @ w1.T, 2.0 * torch.eye(128)[:128, :128], atol=1e-2)
    assert float(parts["first_layer.bias"].abs().max()) > 0
    flat = L.init_flat_rnn_params(1, D_, A_, False)
    assert float(gr.split_net(flat, D_, A_)[7].abs().max()) > 0   # no orthogonal init: final_layer keeps nn.Linear's default


@pytest.mark.parametrize("alg,cls", [("idqn", "QNetwork"), ("vdn", "VDNetwork"), ("qmix", "QMixNetwork")])
def test_config_reaches_recurrent_model(alg, cls):
    from codebase_b200.config import compose

    c = compose([f"+algorithm={alg}", "env.name=lbforaging:Foraging-8x8-2p-3f-v3", "env.time_limit=25", "algorithm.model.use_rnn=True"])
    assert c.algorithm.model._target_ == f"dqn.model.{cls}" and c.algorithm.model.use_rnn is True


def test_library_exports_recurrent_entry_points():
    from codebase_b200 import _native as nat

    lib = nat.lib()
    for name in ("marl_dqn_create_rnn", "marl_dqn_forward_rnn"):
        assert hasattr(lib, name), name

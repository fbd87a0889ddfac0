"""Recurrent (GRU) actor and critic networks of IA2C / IPPO / MAA2C / MAPPO (actor.use_rnn / critic.use_rnn), CPU side: the oracle restatement
(tests/gru_ac_ref.py over oracle/learner_ref.py and oracle/gru_ref.py) against outputs of the reference project's own A2CNetwork / PPONetwork stored
under tests/golden/rnn_ac_*.npz, the host-side parameter layout and key names of the four actor / critic combinations, the initialisation rule,
config composition and the exported symbols.  The device kernels are checked in test_rnn_ac_gpu.py."""
import collections
import math
import os
import types

import numpy as np
import pytest
import torch

from oracle import gru_ref as gr
from oracle import learner_ref as lr
from tests import gru_ac_ref as gar
from tests.helpers import ac_batch, ac_oracle_batch

N, T, P, A = 2, 6, 8, 6
STRIDE = 37   # parameter-sized arrays keep every STRIDE-th element (a prime: the samples fall on every column of the 128-wide rows)
GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
STEPS = (0, 3, 4)   # environment step of each update: hard syncs (interval 2) at 0 and 4, none at 3

# name: (PPO, actor_rnn, critic_rnn, parameter sharing, centralised critic, D, hyper-parameters, standardise_returns, seed)
CASES = {
    "ia2c_indep": (False, True, True, False, False, 9, dict(target_update_interval_or_tau=2.0), False, 201),
    "ia2c_shared_clip_polyak": (False, True, True, True, False, 9, dict(grad_clip=0.5, target_update_interval_or_tau=0.05), False, 202),
    "ippo_indep_clip": (True, True, True, False, False, 9, dict(lr=3e-3, grad_clip=0.5, target_update_interval_or_tau=2.0), False, 203),
    "mappo_shared_central": (True, True, True, True, True, 15, dict(target_update_interval_or_tau=2.0), False, 204),
    "ia2c_standardise": (False, True, True, False, False, 9, dict(target_update_interval_or_tau=2.0), True, 205),
    "ia2c_rnn_actor_mlp_critic": (False, True, False, False, False, 9, dict(target_update_interval_or_tau=2.0), False, 206),
}
EPOCHS = 4
Batch = collections.namedtuple("Batch", ["obss", "actions", "rewards", "dones", "filled", "action_masks"])   # ac/train.py's on-policy batch


def golden_path(name):
    return os.path.join(GOLDEN_DIR, f"rnn_ac_{name}.npz")


def case_setup(name):
    """(hp, D, critic input width, actor_net, critic_net, actor0, critic0, batches (device layout), act-step observations [10][N][D]) of a case;
    parameters and data regenerated from the seed"""
    ppo, arnn, crnn, sharing, central, D, kw, standardise, seed = CASES[name]
    hp = lr.A2CHP(**{**dict(lr=3e-4, gamma=0.99, grad_clip=0.0, n_steps=5, entropy_coef=0.001, value_loss_coef=0.5), **kw})
    nets = [0] * N if sharing else list(range(N))
    n_nets, CD = max(nets) + 1, (N * D if central else D)
    torch.manual_seed(seed)
    actor0 = gar.init_part(arnn, n_nets, D, A)
    critic0 = gar.init_part(crnn, n_nets, CD, 1)
    rng = np.random.default_rng(seed)
    batches = []
    for _ in STEPS:
        s = ac_batch(rng, P, N, T, D, A=A)
        s["obs"] = (s["obs"] / 6.0).astype(np.float32)   # LBF-like magnitudes keep the GRU away from saturation
        batches.append(s)
    act_obs = (rng.integers(-1, 12, size=(10, N, D)) / 6.0).astype(np.float32)
    return hp, D, CD, nets, actor0, critic0, batches, act_obs


def oracle_state(name, actor0, critic0, nets, D):
    ppo, arnn, crnn, sharing, central, _, _, standardise, _ = CASES[name]
    return lr.A2CState(actor0.clone(), critic0.clone(), critic0.clone(), nets, list(nets), D, A, centralised=central,
                       ret_ms=lr.RunningMeanStdRef((N,)) if standardise else None)


def oracle_update(name, st, batch, hp, step):
    if CASES[name][0]:
        return gar.ppo_update(st, batch, hp, step, EPOCHS, 0.2)
    return gar.a2c_update(st, batch, hp, step)


def last_clipped(name, res):
    """the gradient the last optimiser step of an update consumed (after clip_grad_norm_), [actor | critic]"""
    g = res["grads_clipped"][-1] if CASES[name][0] else res["grad_clipped"]
    return torch.cat([g["actor"], g["critic"]])


def make_golden():
    """Regenerates tests/golden/rnn_ac_*.npz from the reference project (MARL_REFERENCE_ROOT): its A2CNetwork / PPONetwork with use_rnn=True on
    the recurrent parts, loaded with each case's parameters, run through three updates, and ten act() / get_value() steps carrying the hiddens."""
    from oracle import ref_shim

    ref = ref_shim.load()
    for name, (ppo, arnn, crnn, sharing, central, D, kw, standardise, seed) in CASES.items():
        hp, D, CD, nets, actor0, critic0, batches, act_obs = case_setup(name)
        cfg = ref_shim.a2c_cfg(standardise_returns=standardise, num_epochs=EPOCHS, ppo_clip=0.2, lr=hp.lr, grad_clip=hp.grad_clip or False,
                               target_update_interval_or_tau=hp.target_update_interval_or_tau)
        anet = types.SimpleNamespace(layers=[128, 128], parameter_sharing=sharing, use_rnn=arnn, use_orthogonal_init=True, centralised=False)
        cnet = types.SimpleNamespace(layers=[128, 128], parameter_sharing=sharing, use_rnn=crnn, use_orthogonal_init=True, centralised=central)
        cls = ref.ac_model.PPONetwork if ppo else ref.ac_model.A2CNetwork
        model = cls([ref_shim.Space(shape=(D,))] * N, [ref_shim.Space(n=A)] * N, cfg, anet, cnet, "cpu")
        kind = "networks" if sharing else "independent"
        n_nets = max(nets) + 1
        sd_of = lambda rnn, flat, prefix, ind, outd: (gr.state_dict_from_flat if rnn else lr.state_dict_from_flat)(flat, prefix, n_nets, ind, outd)  # noqa: E731
        sd = {**sd_of(arnn, actor0, f"actor.{kind}", D, A), **sd_of(crnn, critic0, f"critic.{kind}", CD, 1), **sd_of(crnn, critic0, f"target_critic.{kind}", CD, 1)}
        assert set(sd) == set(model.state_dict()), sorted(set(sd) ^ set(model.state_dict()))[:4]
        model.load_state_dict(sd)
        trained = list(model.actor.parameters()) + list(model.critic.parameters())
        out = dict(stride=np.int32(STRIDE), actor0=actor0.numpy()[::STRIDE], critic0=critic0.numpy()[::STRIDE],
                   **{f"b{u}_{k}": v for u, s in enumerate(batches) for k, v in s.items()})
        # ten consecutive act() / get_value() steps of one env from init_*_hiddens, at the initial parameters
        ah, ch = model.init_actor_hiddens(1), model.init_critic_hiddens(1)
        logits, ahs, values, chs = [], [], [], []
        for s in range(10):
            inputs = [torch.tensor(act_obs[s, a]).view(1, -1) for a in range(N)]
            with torch.no_grad():
                lg, _ = model.actor([x.unsqueeze(0) for x in inputs], ah)
                v, ch = model.get_value([x.unsqueeze(0) for x in inputs], ch)
                _, ah = model.act(inputs, ah)
            logits.append(np.stack([x.reshape(-1).numpy() for x in lg])); values.append(v.reshape(-1).numpy())
            if arnn:
                ahs.append(np.stack([h.reshape(-1).numpy() for h in ah]))
            if crnn:
                chs.append(np.stack([h.reshape(-1).numpy() for h in ch]))
        out.update(act_obs=act_obs, act_logits=np.stack(logits), act_values=np.stack(values))
        if arnn:
            out["act_h"] = np.stack(ahs)
        if crnn:
            out["value_h"] = np.stack(chs)
        metrics = []
        for u, (step, s) in enumerate(zip(STEPS, batches)):
            b = ac_oracle_batch(s)
            res = model.update(Batch(b["obss"], b["actions"], b["rewards"], b["dones"], b["filled"], None), step)
            metrics.append([res[k] for k in ("loss", "actor_loss", "value_loss", "entropy")])
            if u == 0:   # after clip_grad_norm_: the gradient the (last) optimiser step of the first update consumed
                out["grad0"] = torch.cat([p.grad.reshape(-1) for p in trained]).numpy()[::STRIDE]
        out["metrics"] = np.array(metrics, np.float64)
        out["actor3"] = torch.cat([p.data.reshape(-1) for p in model.actor.parameters()]).numpy()[::STRIDE]
        out["critic3"] = torch.cat([p.data.reshape(-1) for p in model.critic.parameters()]).numpy()[::STRIDE]
        out["target3"] = torch.cat([p.data.reshape(-1) for p in model.target_critic.parameters()]).numpy()[::STRIDE]
        out["m3"] = torch.cat([model.optimizer.state[p]["exp_avg"].reshape(-1) for p in trained]).numpy()[::STRIDE]
        out["v3"] = torch.cat([model.optimizer.state[p]["exp_avg_sq"].reshape(-1) for p in trained]).numpy()[::STRIDE]
        if standardise:
            out.update(ret_mean=model.ret_ms.mean.numpy(), ret_var=model.ret_ms.var.numpy(), ret_count=np.float64(model.ret_ms.count))
        np.savez_compressed(golden_path(name), **out)


def _act_steps(flat, nets, obs, ind, outd, central):
    x = torch.tensor(obs).unsqueeze(1)   # (S, E = 1, N, D)
    return gar.act_steps(flat, nets, gar.joint(x) if central else x, ind, outd)


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_reference_golden(name):
    """three updates and ten act() / get_value() steps of the reference's recurrent learner, recorded under tests/golden: the metrics, the first
    update's clipped gradient, Adam m / v, actor, critic, target critic, return statistics, act-step logits / values and hiddens -- all to 1e-5,
    Adam's state and the gradient scaled per tensor"""
    g = np.load(golden_path(name))
    ppo, arnn, crnn, sharing, central, D, kw, standardise, _ = CASES[name]
    hp, D, CD, nets, actor0, critic0, _, _ = case_setup(name)
    assert np.array_equal(actor0.numpy()[::STRIDE], g["actor0"]) and np.array_equal(critic0.numpy()[::STRIDE], g["critic0"]), \
        "the seeded initial parameters differ from the ones the fixture was made from"
    st = oracle_state(name, actor0, critic0, nets, D)
    clip_seen = False
    for u, step in enumerate(STEPS):
        batch = ac_oracle_batch({k: g[f"b{u}_{k}"] for k in ("obs", "act", "rew", "done", "filled")})
        res = oracle_update(name, st, batch, hp, step)
        want = g["metrics"][u]
        got = [res[k] for k in ("loss", "actor_loss", "value_loss", "entropy")]
        np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-5, err_msg=f"metrics of update {u}")
        if ppo:
            clip_seen |= max(res["clip_frac"]) > 0
        if u == 0:
            gc = last_clipped(name, res).numpy()[::STRIDE]
            assert np.abs(gc - g["grad0"]).max() <= 1e-5 * max(1.0, float(np.abs(g["grad0"]).max()))
    for mine, key in ((st.actor, "actor3"), (st.critic, "critic3"), (st.target, "target3")):
        np.testing.assert_allclose(mine.numpy()[::STRIDE], g[key], rtol=0, atol=1e-5, err_msg=key)
    # Adam state per part, relative to each part's scale (v holds squared gradients: twice the gradient's relative error, over three updates)
    na = st.actor.numel()
    for key, mine, tol in (("m3", torch.cat([st.m["actor"], st.m["critic"]]), 2e-5), ("v3", torch.cat([st.v["actor"], st.v["critic"]]), 6e-5)):
        mine = mine.numpy()[::STRIDE]
        cut = len(range(0, na, STRIDE))
        for sl in (slice(0, cut), slice(cut, None)):
            err, scale = float(np.abs(mine[sl] - g[key][sl]).max()), max(float(np.abs(g[key][sl]).max()), 1e-30)
            assert err <= tol * scale, (key, sl, err, scale)
    if standardise:
        np.testing.assert_allclose(st.ret_ms.mean.numpy(), g["ret_mean"], rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(st.ret_ms.var.numpy(), g["ret_var"], rtol=1e-5)
        assert abs(st.ret_ms.count - float(g["ret_count"])) < 1e-9
    if name == "ippo_indep_clip":
        assert clip_seen, "the case is meant to reach the clipped surrogate"
    if arnn:
        q, h = _act_steps(actor0, nets, g["act_obs"], D, A, False)
        np.testing.assert_allclose(q[:, 0].numpy(), g["act_logits"], rtol=0, atol=1e-5)
        np.testing.assert_allclose(h[:, 0].numpy(), g["act_h"], rtol=0, atol=1e-5)
    if crnn:
        v, h = _act_steps(critic0, nets, g["act_obs"], CD, 1, central)
        np.testing.assert_allclose(v[:, 0, :, 0].numpy(), g["act_values"], rtol=0, atol=1e-5)
        np.testing.assert_allclose(h[:, 0].numpy(), g["value_h"], rtol=0, atol=1e-5)


def test_fixtures_stay_small():
    assert sum(os.path.getsize(golden_path(n)) for n in CASES) < 3 << 20


# ---- host-side layout, key names, initialisation -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("arnn,crnn", [(False, False), (True, False), (False, True), (True, True)])
def test_layout_tables_and_key_names(arnn, crnn):
    """the flat [actor | critic] layout and the reference's state_dict names of each part, for the four combinations (shared actor, independent
    centralised critic)"""
    from codebase_b200 import learner as L

    D_, CD = 15, 30
    na, nc = (gr.net_size(D_, A) if arnn else lr.net_size(D_, A)), 2 * (gr.net_size(CD, 1) if crnn else lr.net_size(CD, 1))
    assert gr.net_size(15, 6) == 101_894 and gr.net_size(30, 1) == 103_169
    flat = torch.randn(na + nc)
    shapes_a = (L.rnn_shapes if arnn else L.mlp_shapes)(D_, A)
    shapes_c = (L.rnn_shapes if crnn else L.mlp_shapes)(CD, 1)
    sd = {**L.flat_to_state_dict(flat[:na], "actor.networks", 1, shapes_a), **L.flat_to_state_dict(flat[na:], "critic.independent", 2, shapes_c)}
    first_a = "actor.networks.0.first_layer.weight" if arnn else "actor.networks.0.network.0.weight"
    first_c = "critic.independent.1.rnn.weight_hh_l0" if crnn else "critic.independent.1.network.2.weight"
    assert first_a in sd and first_c in sd and tuple(sd[first_c].shape) == ((384, 128) if crnn else (128, 128))
    if arnn:
        assert list(sd)[:8] == [f"actor.networks.0.{n}" for n in gr.NAMES]
    back_a = L.state_dict_to_flat(sd, "actor.networks", 1, shapes_a)
    back_c = L.state_dict_to_flat(sd, "critic.independent", 2, shapes_c)
    assert torch.equal(torch.cat([back_a, back_c]), flat)
    assert gar.is_recurrent(flat[:na], [0, 0], D_, A) == arnn and gar.is_recurrent(flat[na:], [0, 1], CD, 1) == crnn


def test_host_initialisation_rule():
    """a recurrent part: orthogonal (gain sqrt 2, zero bias) on final_layer only, PyTorch's defaults elsewhere; an MLP part: orthogonal on every layer"""
    from codebase_b200 import learner as L

    torch.manual_seed(4)
    parts = dict(zip(gr.NAMES, gr.split_net(L.init_flat_rnn_params(1, 30, 1, True), 30, 1)))
    w3 = parts["final_layer.weight"]
    assert torch.allclose(w3 @ w3.T, 2.0 * torch.eye(1), atol=1e-5) and torch.all(parts["final_layer.bias"] == 0)
    bound = 1 / math.sqrt(128)
    for k in ("rnn.weight_ih_l0", "rnn.weight_hh_l0", "rnn.bias_ih_l0", "rnn.bias_hh_l0"):
        assert 0.9 * bound < float(parts[k].abs().max()) <= bound, k
    assert float(parts["first_layer.weight"].abs().max()) <= 1 / math.sqrt(30) and float(parts["first_layer.bias"].abs().max()) > 0
    w1, b1 = lr.split_net(L.init_flat_params(1, 15, 6, True), 15, 6)[:2]
    assert torch.allclose(w1.T @ w1, 2.0 * torch.eye(15), atol=1e-4) and torch.all(b1 == 0)


@pytest.mark.parametrize("alg,cls", [("ia2c", "A2CNetwork"), ("ippo", "PPONetwork"), ("maa2c", "A2CNetwork"), ("mappo", "PPONetwork")])
@pytest.mark.parametrize("flags", [(True, True), (True, False), (False, True)])
def test_config_reaches_recurrent_model(alg, cls, flags):
    from codebase_b200.config import compose

    over = [f"algorithm.model.actor.use_rnn={flags[0]}", f"algorithm.model.critic.use_rnn={flags[1]}"]
    c = compose([f"+algorithm={alg}", "env.name=lbforaging:Foraging-8x8-2p-3f-v3", "env.time_limit=25", *over])
    m = c.algorithm.model
    assert m._target_ == f"ac.model.{cls}" and m.actor.use_rnn is flags[0] and m.critic.use_rnn is flags[1]


def test_library_exports_recurrent_entry_points():
    from codebase_b200 import _native as nat

    lib = nat.lib()
    for name in ("marl_a2c_create_rnn", "marl_a2c_forward_rnn"):
        assert hasattr(lib, name), name

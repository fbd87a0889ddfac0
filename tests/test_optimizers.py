"""algorithm.optimizer (CPU): the oracle's optimiser steps (tests/optim_ref.py) against torch.optim itself, the name / class parsing of the
host, and the refusal of every other torch.optim optimiser before any native call."""
import dataclasses
import types

import pytest
import torch

from tests import optim_ref as orf
from tests.helpers import space

TORCH_CLASS = {"Adam": torch.optim.Adam, "AdamW": torch.optim.AdamW, "RMSprop": torch.optim.RMSprop, "Adagrad": torch.optim.Adagrad,
               "SGD": torch.optim.SGD}


@pytest.mark.parametrize("name", orf.NAMES)
@pytest.mark.parametrize("lr", [3e-4, 1e-2])
def test_oracle_step_is_torch_optim_bitwise(name, lr):
    """20 steps on random gradients of widely spread magnitude: parameters and every state tensor equal torch.optim.<name>(lr=lr) bit for bit
    (torch's CPU tensors take the single-tensor path, as in the reference)"""
    g = torch.Generator().manual_seed(11)
    p = torch.nn.Parameter(torch.randn(4099, generator=g))
    opt = TORCH_CLASS[name]([p], lr=lr)
    theta, m, v = p.detach().clone(), torch.zeros(4099), torch.zeros(4099)
    for step in range(1, 21):
        grad = torch.randn(4099, generator=g) * torch.exp(torch.randn(4099, generator=g) * 4)
        grad[::97] = 0.0
        p.grad = grad.clone()
        opt.step()
        orf.STEPS[name](theta, m, v, grad, step, lr)
        assert torch.equal(theta, p.detach()), (name, step, float((theta - p.detach()).abs().max()))
        state = opt.state[p]
        for buf, key in zip((m, v), orf.STATE[name]):
            if key is None:
                assert not torch.any(buf)
            else:
                assert torch.equal(buf, state[key]), (name, step, key)


def test_context_restores_adam():
    from oracle import learner_ref as lr

    with orf.optimizer("RMSprop"):
        assert lr.adam_step is orf.rmsprop_step
    assert lr.adam_step is orf.STEPS["Adam"]


@pytest.mark.parametrize("name", ["RMSprop", "Adagrad", "SGD"])
def test_device_step_formula_rounds_as_torch(name):
    """opt_step<OPT> (csrc/learner_kernels.cu) restated in float32 with an exact fused multiply-add, with the scalars the host passes
    (set_step_consts), on 200 000 elements over 3 steps: RMSprop's square_avg and Adagrad's sum (addcmul_ = fma(value * g, g, self)) and SGD's
    parameters (add_(alpha=) = fma) equal torch.optim's bit for bit"""
    import numpy as np

    f = np.float32

    def fma(a, b, c):   # a * b is exact in double; then one rounding of the sum to float
        return (np.float64(1) * a * b + c).astype(f)

    g0 = torch.Generator().manual_seed(5)
    p = torch.nn.Parameter(torch.randn(200_000, generator=g0))
    lr = 3e-4
    th, v = p.detach().numpy().copy(), np.zeros(200_000, f)
    opt = TORCH_CLASS[name]([p], lr=lr)
    for step in range(1, 4):
        grad = torch.randn(200_000, generator=g0) * torch.exp(torch.randn(200_000, generator=g0) * 2)
        p.grad = grad.clone()
        opt.step()
        g = grad.numpy()
        if name == "SGD":
            th = fma(f(-lr), g, th)
            assert np.array_equal(th, p.detach().numpy()), step
        else:
            v = fma(g, g, v) if name == "Adagrad" else fma((f(1.0 - 0.99) * g).astype(f), g, (v * f(0.99)).astype(f))
            assert np.array_equal(v, opt.state[p][orf.STATE[name][1]].numpy()), step


# ---- the host's parsing ----------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("value,name", [("Adam", "Adam"), ("AdamW", "AdamW"), ("RMSprop", "RMSprop"), ("Adagrad", "Adagrad"), ("SGD", "SGD"),
                                        (torch.optim.Adam, "Adam"), (torch.optim.AdamW, "AdamW"), (torch.optim.RMSprop, "RMSprop"),
                                        (torch.optim.Adagrad, "Adagrad"), (torch.optim.SGD, "SGD")])
def test_names_and_classes_parse(value, name):
    from codebase_b200 import optimizers

    assert optimizers.optimizer_name(value) == name


REFUSED = ["Adamax", "NAdam", "RAdam", "Adadelta", "ASGD", "Rprop", "LBFGS", "SparseAdam", "Adafactor", "adam", "rmsprop", "Muon"]


@pytest.mark.parametrize("name", REFUSED)
def test_other_optimizers_are_refused(name):
    from codebase_b200 import optimizers

    msg = r"is not implemented; the GPU learners implement Adam, AdamW, RMSprop, Adagrad, SGD"
    with pytest.raises(NotImplementedError, match=msg):
        optimizers.optimizer_name(name)
    cls = getattr(torch.optim, name, None)
    if isinstance(cls, type):
        with pytest.raises(NotImplementedError, match=msg):
            optimizers.optimizer_name(cls)


def test_native_constants_are_torch_defaults():
    """the marl_optimizer of each name carries torch's defaults (lr comes from algorithm.lr)"""
    import inspect

    from codebase_b200 import optimizers

    for name, cls in TORCH_CLASS.items():
        o = optimizers.native(name)
        d = {k: v.default for k, v in inspect.signature(cls.__init__).parameters.items()}
        assert o.kind == optimizers.SUPPORTED.index(name)
        if "betas" in d and name in ("Adam", "AdamW"):
            assert (o.beta1, o.beta2) == pytest.approx(d["betas"], rel=1e-7)
        if name in ("Adam", "AdamW", "RMSprop", "Adagrad"):
            assert o.eps == pytest.approx(d["eps"], rel=1e-7)
        if name == "RMSprop":
            assert o.alpha == pytest.approx(d["alpha"], rel=1e-7)
        assert o.weight_decay == pytest.approx(d.get("weight_decay", 0.0) if name == "AdamW" else 0.0, rel=1e-7)
        for zero in ("momentum", "lr_decay", "initial_accumulator_value"):
            assert d.get(zero, 0) in (0, 0.0), (name, zero)
        assert not d.get("amsgrad", False) and not d.get("nesterov", False) and not d.get("centered", False) and not d.get("maximize", False)


def _net(**kw):
    return types.SimpleNamespace(layers=[128, 128], parameter_sharing=False, use_rnn=False, use_orthogonal_init=True, centralised=False, **kw)


@pytest.mark.parametrize("family", ["QNetwork", "VDNetwork", "QMixNetwork", "A2CNetwork", "PPONetwork"])
@pytest.mark.parametrize("opt", ["NAdam", torch.optim.Adamax])
def test_refusal_comes_before_any_native_call(family, opt, monkeypatch):
    from codebase_b200 import _native as nat
    from codebase_b200.ac import model as AM
    from codebase_b200.dqn import model as DM

    def no_lib():
        raise AssertionError("the native library was reached")

    monkeypatch.setattr(nat, "lib", no_lib)
    obs, act = [space(shape=(11,))] * 2, [space(n=6)] * 2
    if family in ("A2CNetwork", "PPONetwork"):
        cfg = types.SimpleNamespace(optimizer=opt, lr=3e-4, gamma=0.99, grad_clip=0.0, n_steps=5, entropy_coef=0.001, value_loss_coef=0.5,
                                    target_update_interval_or_tau=200, standardise_returns=False, num_epochs=4, ppo_clip=0.2)
        make = lambda: getattr(AM, family)(obs, act, cfg, _net(), _net(), "cuda")   # noqa: E731
    else:
        cfg = types.SimpleNamespace(optimizer=opt, lr=3e-4, gamma=0.99, grad_clip=1.0, double_q=False, target_update_interval_or_tau=200,
                                    standardise_returns=False)
        args = (obs, act, cfg, [128, 128], False, False, True)
        if family == "QMixNetwork":
            make = lambda: DM.QMixNetwork(*args, dict(embed_dim=32, hypernet_layers=2, hypernet_embed=64), "cuda")   # noqa: E731
        else:
            make = lambda: getattr(DM, family)(*args, "cuda")   # noqa: E731
    with pytest.raises(NotImplementedError, match=r"Adam, AdamW, RMSprop, Adagrad, SGD"):
        make()


def test_cli_accepts_rmsprop_for_every_overlay():
    """algorithm.optimizer=RMSprop composes for all seven overlays, which keep "Adam" as their default"""
    from codebase_b200.config import compose

    for algo in ("idqn", "vdn", "qmix", "ia2c", "ippo", "maa2c", "mappo"):
        base = ["+algorithm=" + algo, "env.name=lbforaging:Foraging-8x8-2p-3f-v3", "env.time_limit=25"]
        assert compose(base).algorithm.optimizer == "Adam"
        assert compose(base + ["algorithm.optimizer=RMSprop"]).algorithm.optimizer == "RMSprop"


# ---- the oracle learners against the reference's classes with each optimiser (tests/golden/optimizers_reference.npz) ------------------------------
@dataclasses.dataclass(frozen=True)
class RefCase:
    fam: str               # the reference's class
    N: int = 2
    D: int = 15
    sharing: bool = False
    seed: int = 0
    rnn: bool = False      # GRU agent networks (DQN) / GRU actor and critic (actor-critic)
    central: bool = False  # centralised critic
    grad_clip: float = 0.0
    obs_scale: float = 1.0


# 3 updates of each with every optimiser besides Adam.  QMIX: observations / 10 (at full scale the unclipped mixer's first SGD step diverges, in
# the reference as here); recurrent cases: / 6, LBF-like magnitudes that keep the GRU away from saturation (tests/test_rnn_dqn.py)
REF_CASES = {
    "idqn": RefCase("QNetwork", seed=61, grad_clip=1.0),
    "vdn_shared": RefCase("VDNetwork", sharing=True, seed=62, grad_clip=1.0),
    "qmix": RefCase("QMixNetwork", seed=65, grad_clip=1.0, obs_scale=0.1),   # two-layer hypernetworks (embed 64, hypernet_embed 32)
    "idqn_rnn": RefCase("QNetwork", seed=66, rnn=True, grad_clip=1.0, obs_scale=1 / 6),
    "ia2c": RefCase("A2CNetwork", seed=63),
    "maa2c": RefCase("A2CNetwork", seed=67, central=True),
    "mappo": RefCase("PPONetwork", seed=64, central=True, grad_clip=0.5),   # 4 epochs
    "ia2c_rnn": RefCase("A2CNetwork", seed=68, rnn=True, obs_scale=1 / 6),
}
OPTS = ("AdamW", "RMSprop", "Adagrad", "SGD")
REF_T, REF_B, REF_A, REF_UPDATES, REF_EPOCHS = 10, 16, 6, 3, 4
MIXING = dict(embed_dim=64, hypernet_layers=2, hypernet_embed=32)
# parameter-sized vectors: every 127th element (MLP) / 1021st (GRU: 5x the parameters); primes, so that rows of 128 are not always sampled in
# the same column.  Eight cases x 4 optimisers x 3 updates of 5 vectors stay under 1 MB.
STRIDE_MLP, STRIDE_RNN = 127, 1021


def is_dqn(c):
    return c.fam in ("QNetwork", "VDNetwork", "QMixNetwork")


def _ref_case(key):
    """(oracle state, hyper-parameters) a case starts from"""
    from oracle import gru_ref as gr
    from oracle import learner_ref as lr
    from oracle import qmix_ref as qr
    from tests import gru_ac_ref as gar
    from tests.helpers import seeded_params

    c = REF_CASES[key]
    n_nets, nets = (1, [0] * c.N) if c.sharing else (c.N, list(range(c.N)))
    if is_dqn(c):
        torch.manual_seed(c.seed)
        theta = gr.init_flat(n_nets, c.D, REF_A) if c.rnn else seeded_params(lr, n_nets, c.D, REF_A, c.seed)
        hp = lr.DqnHP(grad_clip=c.grad_clip, double_q=True, target_update_interval_or_tau=2, mixer=min(1, ("QNetwork", "VDNetwork", "QMixNetwork").index(c.fam)))
        if c.fam == "QMixNetwork":
            mix = qr.init_mixer_flat(c.N, c.N * c.D, MIXING["embed_dim"], MIXING["hypernet_embed"])
            st = qr.QmixState(theta.clone(), theta.clone(), mix.clone(), mix.clone(), nets, c.D, REF_A, MIXING["embed_dim"], MIXING["hypernet_embed"])
        else:
            st = lr.DqnState(theta.clone(), theta.clone(), nets, c.D, REF_A)
    else:
        CD = c.N * c.D if c.central else c.D
        if c.rnn:
            torch.manual_seed(c.seed)
            actor, critic = gar.init_part(True, n_nets, c.D, REF_A), gar.init_part(True, n_nets, CD, 1)
        else:
            actor, critic = seeded_params(lr, n_nets, c.D, REF_A, c.seed), seeded_params(lr, n_nets, CD, 1, c.seed + 1)
        st = lr.A2CState(actor, critic.clone(), critic.clone(), nets, nets, c.D, REF_A, centralised=c.central)
        hp = lr.A2CHP(grad_clip=c.grad_clip, target_update_interval_or_tau=2)
    return st, hp


def _ref_batches(key):
    """(oracle batch, device-layout store, replay indices or None) per update"""
    import numpy as np

    from oracle import learner_ref as lr
    from tests.helpers import ac_batch, ac_oracle_batch, random_store

    c = REF_CASES[key]
    rng = np.random.default_rng(c.seed)
    out = []
    for _ in range(REF_UPDATES):
        if is_dqn(c):
            s = random_store(rng, 64, c.N, REF_T, c.D, c.fam != "QNetwork")
            s["obs"] = (s["obs"] * np.float32(c.obs_scale)).astype(np.float32)
            idx = rng.integers(0, 64, size=REF_B)
            out.append((lr.batch_from_store(s, idx), s, idx))
        else:
            s = ac_batch(rng, REF_B, c.N, REF_T, c.D)
            s["obs"] = (s["obs"] * np.float32(c.obs_scale)).astype(np.float32)
            out.append((ac_oracle_batch(s), s, None))
    return out


def _flat_parts(st, c):
    """(trained parameters, their target, m, v) of an oracle state, flat in the order of the reference's optimiser: DQN the agents' networks
    (QMIX: then the mixer), actor-critic the actor then the critic; the targets in the same order"""
    if is_dqn(c):
        if c.fam == "QMixNetwork":
            return (torch.cat([st.theta, st.mix]), torch.cat([st.theta_tgt, st.mix_tgt]), torch.cat([st.m, st.mix_m]), torch.cat([st.v, st.mix_v]))
        return st.theta.clone(), st.theta_tgt.clone(), st.m.clone(), st.v.clone()
    return (torch.cat([st.actor, st.critic]), st.target.clone(), torch.cat([st.m["actor"], st.m["critic"]]), torch.cat([st.v["actor"], st.v["critic"]]))


def run_oracle(key, opt):
    """the oracle (with optimiser `opt`) over the case's updates: per update dict(loss, grad = the gradient the optimiser consumed (after the
    clip), theta, target, m, v), flat as _flat_parts"""
    from oracle import gru_ref as gr
    from oracle import learner_ref as lr
    from tests import gru_ac_ref as gar

    c = REF_CASES[key]
    st, hp = _ref_case(key)
    rec = []
    for u, (b, _, _) in enumerate(_ref_batches(key)):
        with orf.optimizer(opt):
            if c.fam == "QMixNetwork":
                res = orf.qmix_update(st, b, hp, opt)
                g = res["grad"] * lr.clip_coef(res["grad"], hp.grad_clip)[0] if hp.grad_clip else res["grad"]
                grad = torch.cat([g, res["mix_grad"]])
            elif is_dqn(c):
                res = gr.dqn_update(st, b, hp) if c.rnn else lr.dqn_update(st, b, hp)
                grad = res["grad_clipped"]
            elif c.fam == "PPONetwork":
                res = (gar.ppo_update if c.rnn else lr.ppo_update)(st, b, hp, u, REF_EPOCHS, 0.2)
                grad = torch.cat([res["grads_clipped"][-1]["actor"], res["grads_clipped"][-1]["critic"]])
            else:
                res = (gar.a2c_update if c.rnn else lr.a2c_update)(st, b, hp, u)
                grad = torch.cat([res["grad_clipped"]["actor"], res["grad_clipped"]["critic"]])
        theta, tgt, m, v = _flat_parts(st, c)
        rec.append(dict(loss=res["loss"], grad=grad.detach().clone(), theta=theta.clone(), target=tgt.clone(), m=m.clone(), v=v.clone()))
    return rec


def fixture_stride(key):
    return STRIDE_RNN if REF_CASES[key].rnn else STRIDE_MLP


@pytest.mark.parametrize("opt", OPTS)
@pytest.mark.parametrize("key", list(REF_CASES))
def test_oracle_matches_reference(key, opt):
    """oracle learners with each optimiser vs what the reference's QNetwork / VDNetwork / QMixNetwork / A2CNetwork / PPONetwork (MLP and GRU)
    computed with torch.optim.<opt>: loss, clipped gradient, parameters, optimiser state and target after every update"""
    import numpy as np

    from tests.helpers import reference_outputs

    g = reference_outputs("optimizers_reference")
    stride = int(g[f"{key}_stride"])
    # one thread, as the fixture was made (a reduction split over threads rounds differently)
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        rec = run_oracle(key, opt)
    finally:
        torch.set_num_threads(threads)
    # optimiser state relative to its largest element: 2e-5 (v ~ g^2 doubles the gradient's 1e-5); recurrent cases 5e-5, as the oracle's GRU
    # gradient agrees with the reference's to ~2e-5 of its scale (tests/test_rnn_dqn.py compares Adam's m at 3e-5)
    stol = 5e-5 if REF_CASES[key].rnn else 2e-5
    for u, r in enumerate(rec):
        p = f"{key}_{opt}_{u}"
        assert abs(r["loss"] - float(g[f"{p}_loss"])) <= 1e-5 * max(1.0, abs(r["loss"])), (p, r["loss"], float(g[f"{p}_loss"]))
        want = g[f"{p}_grad"]
        assert np.abs(r["grad"].numpy()[::stride] - want).max() <= 1e-5 * max(1.0, float(np.abs(want).max())), (p, "grad")
        for name in ("theta", "target"):
            d = np.abs(r[name].numpy()[::stride] - g[f"{p}_{name}"])
            assert np.quantile(d, 0.999) < 1e-5, (p, name, d.max())
        for name, buf in zip(orf.STATE[opt], (r["m"], r["v"])):
            if name is not None:
                want = g[f"{p}_{name}"]
                assert np.abs(buf.numpy()[::stride] - want).max() <= stol * max(float(np.abs(want).max()), 1e-30), (p, name)


def make_reference_outputs(ref, ref_shim):
    """tests/golden/optimizers_reference.npz: the reference's learner classes, built with cfg.optimizer = each of OPTS, on REF_CASES"""
    import os
    import types as T
    from collections import namedtuple

    import numpy as np

    from oracle import gru_ref as gr
    from oracle import learner_ref as lr
    from oracle import qmix_ref as qr
    from tests.helpers import GOLDEN

    ABatch = namedtuple("Batch", ["obss", "actions", "rewards", "dones", "filled", "action_masks"])
    out = {}
    for key, c in REF_CASES.items():
        stride = fixture_stride(key)
        out[f"{key}_stride"] = np.int64(stride)
        kind, n_nets = ("networks", 1) if c.sharing else ("independent", c.N)
        CD = c.N * c.D if c.central else c.D
        sd_of = gr.state_dict_from_flat if c.rnn else lr.state_dict_from_flat
        for opt in OPTS:
            st, hp = _ref_case(key)
            spaces = ([ref_shim.Space(shape=(c.D,))] * c.N, [ref_shim.Space(n=REF_A)] * c.N)
            if is_dqn(c):
                cfg = ref_shim.dqn_cfg(optimizer=opt, target_update_interval_or_tau=2, grad_clip=c.grad_clip or False)
                args = (*spaces, cfg, [128, 128], c.sharing, c.rnn, True)
                model = (ref.dqn_model.QMixNetwork(*args, MIXING, "cpu") if c.fam == "QMixNetwork" else getattr(ref.dqn_model, c.fam)(*args, "cpu"))
                sd = {**sd_of(st.theta, f"critic.{kind}", n_nets, c.D, REF_A), **sd_of(st.theta_tgt, f"target.{kind}", n_nets, c.D, REF_A)}
                params, tparams = list(model.critic.parameters()), list(model.target.parameters())
                if c.fam == "QMixNetwork":
                    E, He = MIXING["embed_dim"], MIXING["hypernet_embed"]
                    sd.update(qr.mixer_state_dict_from_flat(st.mix, "mixer", c.N, c.N * c.D, E, He))
                    sd.update(qr.mixer_state_dict_from_flat(st.mix_tgt, "target_mixer", c.N, c.N * c.D, E, He))
                    params, tparams = params + list(model.mixer.parameters()), tparams + list(model.target_mixer.parameters())
            else:
                cfg = ref_shim.a2c_cfg(optimizer=opt, grad_clip=c.grad_clip or False, target_update_interval_or_tau=2, num_epochs=REF_EPOCHS, ppo_clip=0.2)
                net = T.SimpleNamespace(layers=[128, 128], parameter_sharing=c.sharing, use_rnn=c.rnn, use_orthogonal_init=True, centralised=False)
                cnet = T.SimpleNamespace(**{**vars(net), "centralised": c.central})
                model = getattr(ref.ac_model, c.fam)(*spaces, cfg, net, cnet, "cpu")
                sd = {**sd_of(st.actor, f"actor.{kind}", n_nets, c.D, REF_A), **sd_of(st.critic, f"critic.{kind}", n_nets, CD, 1),
                      **sd_of(st.target, f"target_critic.{kind}", n_nets, CD, 1)}
                params, tparams = list(model.actor.parameters()) + list(model.critic.parameters()), list(model.target_critic.parameters())
            missing = set(sd) - set(model.state_dict())
            assert not missing, sorted(missing)[:4]
            model.load_state_dict(sd, strict=False)
            flat = lambda ts: torch.cat([t.detach().reshape(-1) for t in ts]).float().numpy()[::stride]   # noqa: E731
            for u, (b, _, _) in enumerate(_ref_batches(key)):
                if is_dqn(c):
                    res = model.update(ref.dqn_train.Batch(b["obss"], b["actions"], b["rewards"], b["dones"], b["filled"], None))
                else:
                    res = model.update(ABatch(b["obss"], b["actions"], b["rewards"], b["dones"].bool(), b["filled"], None), u)
                p = f"{key}_{opt}_{u}"
                out[f"{p}_loss"] = np.float64(res["loss"])
                out[f"{p}_grad"] = flat([q.grad for q in params])   # after clip_grad_norm_: what the (last) optimiser step consumed
                out[f"{p}_theta"] = flat(params)
                out[f"{p}_target"] = flat(tparams)
                for name in orf.STATE[opt]:
                    if name is not None:
                        out[f"{p}_{name}"] = flat([model.optimizer.state[q][name] for q in params])
    np.savez_compressed(os.path.join(GOLDEN, "optimizers_reference.npz"), **out)


if __name__ == "__main__":
    from oracle import ref_shim

    torch.set_num_threads(1)
    make_reference_outputs(ref_shim.load(), ref_shim)

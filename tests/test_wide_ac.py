"""Actor-critic inputs wider than 32 features (up to 128): the host-side width check, and the oracle (oracle.learner_ref) against what the
reference's own A2CNetwork / PPONetwork computed at those widths (tests/golden/wide_ac_reference.npz): MAA2C / MAPPO with 4 agents of 27 features
(a centralised critic of 108 inputs, as on Foraging-15x15-4p-5f-v3) with shared and independent critics, and IA2C at 45 features.

`MARL_REFERENCE_ROOT=<reference checkout> python -m tests.test_wide_ac` regenerates the fixture."""
import os
import types

import numpy as np
import pytest
import torch

from oracle import learner_ref as lr
from tests.helpers import GOLDEN, STRIDE, ac_batch, ac_oracle_batch, load_params, reference_outputs, seeded_params, space

T, A = 25, 6
METRICS = ("loss", "actor_loss", "value_loss", "entropy")
# key: (class, agents N, features D, seed, batch seed, envs P, steps, grad_clip, parameter sharing, centralised critic)
REF_CASES = {
    "maa2c_shared": ("A2CNetwork", 4, 27, 21, 31, 8, (0, 2), False, True, True),
    "maa2c_indep": ("A2CNetwork", 4, 27, 22, 32, 8, (0, 2), False, False, True),
    "mappo_shared": ("PPONetwork", 4, 27, 23, 33, 8, (0, 2), 0.5, True, True),
    "mappo_indep": ("PPONetwork", 4, 27, 24, 34, 8, (0, 2), False, False, True),
    "ia2c_D45": ("A2CNetwork", 2, 45, 25, 35, 8, (0, 2, 3), False, False, False),
}
EPOCHS = 3


def case_state(key):
    """the oracle state a case starts from: seeded weights (actor, critic; the target critic is a copy of the critic)"""
    cls, N, D, seed, _, _, _, clip, sharing, centralised = REF_CASES[key]
    n_nets, nets = (1, [0] * N) if sharing else (N, list(range(N)))
    actor, critic = seeded_params(lr, n_nets, D, A, seed), seeded_params(lr, n_nets, N * D if centralised else D, 1, seed + 1)
    return lr.A2CState(actor, critic.clone(), critic.clone(), nets, nets, D, A, centralised=centralised)


def case_hp(key):
    clip = REF_CASES[key][7]
    return lr.A2CHP(grad_clip=float(clip or 0.0), target_update_interval_or_tau=2)


def case_batches(key):
    """the case's batches in the device layout (numpy), one per update"""
    _, N, D, _, bseed, P, steps, _, _, _ = REF_CASES[key]
    rng = np.random.default_rng(bseed)
    return [ac_batch(rng, P, N, T, D) for _ in steps]


def _close(a, b, rtol=1e-5, atol=1e-5):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert np.allclose(a, b, rtol=rtol, atol=atol), float(np.abs(a - b).max())


@pytest.mark.parametrize("key", list(REF_CASES))
def test_oracle_matches_reference_at_wide_inputs(key):
    """oracle.learner_ref from the case's seeded weights and batches vs what the reference computed for them: losses after every update, actor /
    critic / target parameters after the last"""
    g = reference_outputs("wide_ac_reference")
    cls, _, _, _, _, _, steps, _, _, _ = REF_CASES[key]
    st, hp = case_state(key), case_hp(key)
    metrics = []
    for step, s in zip(steps, case_batches(key)):
        b = ac_oracle_batch(s)
        got = lr.ppo_update(st, b, hp, step, EPOCHS, 0.2) if cls == "PPONetwork" else lr.a2c_update(st, b, hp, step)
        metrics.append([got[k] for k in METRICS])
    _close(metrics, g[f"{key}_metrics"])
    for mine, name in ((st.actor, "actor"), (st.critic, "critic"), (st.target, "target")):
        d = np.abs(mine.numpy()[::STRIDE] - g[f"{key}_{name}"])
        assert np.quantile(d, 0.999) < 1e-5, (name, d.max())


# ---- the host-side width check ----------------------------------------------------------------------------------------------------------------
def _net(centralised):
    return types.SimpleNamespace(layers=[128, 128], parameter_sharing=False, use_rnn=False, use_orthogonal_init=True, centralised=centralised)


def test_host_check_refuses_inputs_wider_than_128():
    from codebase_b200.ac import model as M

    with pytest.raises(NotImplementedError, match=r"actor's observation is 129 wide.*at most 128"):
        M.check_input_widths([space(shape=(129,))] * 2, _net(False))
    with pytest.raises(NotImplementedError, match=r"critic's observation is 129 wide"):
        M.check_input_widths([space(shape=(129,))], _net(True))   # one agent: the critic reads its own observation
    with pytest.raises(NotImplementedError, match=r"5 x 27 = 135 wide.*at most 128"):
        M.check_input_widths([space(shape=(27,))] * 5, _net(True))
    with pytest.raises(NotImplementedError, match=r"9 x 45 = 405"):
        M.check_input_widths([space(shape=(45,))] * 9, _net(True))


@pytest.mark.parametrize("N,D,central", [(1, 128, False), (2, 128, False), (4, 32, True), (4, 27, True), (9, 45, False), (2, 64, True), (3, 18, True)])
def test_host_check_accepts_up_to_128(N, D, central):
    from codebase_b200.ac import model as M

    M.check_input_widths([space(shape=(D,))] * N, _net(central))


@pytest.mark.parametrize("cls", ["A2CNetwork", "PPONetwork"])
def test_constructor_refuses_before_any_native_call(cls, monkeypatch):
    """the check runs first in A2CNetwork.__init__: no device and no library are needed to be refused"""
    from codebase_b200 import _native as nat
    from codebase_b200.ac import model as M

    def no_lib():
        raise AssertionError("the native library was reached")

    monkeypatch.setattr(nat, "lib", no_lib)
    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=0.0, n_steps=5, entropy_coef=0.001, value_loss_coef=0.5,
                                target_update_interval_or_tau=200, standardise_returns=False, num_epochs=4, ppo_clip=0.2)
    with pytest.raises(NotImplementedError, match=r"5 x 27 = 135"):
        getattr(M, cls)([space(shape=(27,))] * 5, [space(n=6)] * 5, cfg, _net(False), _net(True), "cuda")
    with pytest.raises(NotImplementedError, match=r"actor's observation is 129 wide"):
        getattr(M, cls)([space(shape=(129,))] * 2, [space(n=6)] * 2, cfg, _net(False), _net(False), "cuda")


def make_reference_outputs(ref, ref_shim):
    """tests/golden/wide_ac_reference.npz: the reference's A2CNetwork / PPONetwork run on REF_CASES."""
    from collections import namedtuple

    Batch = namedtuple("Batch", ["obss", "actions", "rewards", "dones", "filled", "action_masks"])
    out = {}
    for key, (cls, N, D, _, _, _, steps, clip, sharing, centralised) in REF_CASES.items():
        st = case_state(key)
        cfg = ref_shim.a2c_cfg(grad_clip=clip, num_epochs=EPOCHS, ppo_clip=0.2, target_update_interval_or_tau=2)
        model = getattr(ref.ac_model, cls)([ref_shim.Space(shape=(D,))] * N, [ref_shim.Space(n=A)] * N, cfg, ref_shim.net_cfg(parameter_sharing=sharing),
                                           ref_shim.net_cfg(parameter_sharing=sharing, centralised=centralised), "cpu")
        kind, n_nets = ("networks", 1) if sharing else ("independent", N)
        load_params(model, lr, (f"actor.{kind}",), st.actor, n_nets, D, A)
        load_params(model, lr, (f"critic.{kind}", f"target_critic.{kind}"), st.critic, n_nets, N * D if centralised else D, 1)
        metrics = []
        for step, s in zip(steps, case_batches(key)):
            b = ac_oracle_batch(s)
            want = model.update(Batch(b["obss"], b["actions"], b["rewards"], b["dones"].bool(), b["filled"], None), step)
            metrics.append([float(want[k]) for k in METRICS])
        out[f"{key}_metrics"] = np.array(metrics, np.float64)
        sd = model.state_dict()
        for name, prefix in (("actor", f"actor.{kind}"), ("critic", f"critic.{kind}"), ("target", f"target_critic.{kind}")):
            out[f"{key}_{name}"] = lr.flat_from_state_dict(sd, prefix, n_nets).numpy()[::STRIDE]
    np.savez_compressed(os.path.join(GOLDEN, "wide_ac_reference.npz"), **out)


if __name__ == "__main__":
    from oracle import ref_shim

    torch.set_num_threads(1)
    make_reference_outputs(ref_shim.load(), ref_shim)

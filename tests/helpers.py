"""Shared helpers of the parity tests."""
import functools
import os
import types

import numpy as np
import pytest
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# Parameter-sized vectors that the reference project produced are stored as every STRIDE-th element (fixtures stay small); inputs are stored whole
# or regenerated from seeds.
STRIDE = 8


def reference_outputs(name):
    """What the reference project (marlbase) computed for a test's seeded inputs: tests/golden/<name>.npz, written by tests/golden/make_golden.py."""
    return np.load(os.path.join(GOLDEN, f"{name}.npz"))


def golden_stride(g):
    """stride of the parameter-sized outputs of a fixture (1: stored whole)"""
    return int(g["stride"]) if "stride" in g.files else 1


def seeded_params(lr, n_nets, in_dim, out_dim, seed):
    """Initial weights of a parity case (the reference's orthogonal initialisation, seeded): the tests start the oracle from them, and
    tests/golden/make_golden.py loaded the same weights into the reference model before recording its outputs."""
    return lr.init_flat(n_nets, in_dim, out_dim, generator=torch.Generator().manual_seed(seed))


def load_params(model, lr, prefixes, flat, n_nets, in_dim, out_dim):
    """Copy flat weights into the sub-networks `prefixes` of a reference model (fixture generation only)."""
    sd = {}
    for prefix in prefixes:
        sd.update(lr.state_dict_from_flat(flat, prefix, n_nets, in_dim, out_dim))
    missing = set(sd) - set(model.state_dict())
    assert not missing, sorted(missing)[:4]
    model.load_state_dict(sd, strict=False)

def space(shape=None, n=None):
    """the two gymnasium space kinds the learners read (.shape of a Box, .n of a Discrete)"""
    return types.SimpleNamespace(shape=shape, n=n)


def random_store(rng, cap, N, T, D, coop, A=6):
    """A trajectory store of `cap` random episodes in the device layout (numpy arrays): ragged lengths, sparse rewards (`coop`: agent 0's reward
    for every agent, as CooperativeReward leaves it), most episodes ending in a terminal step."""
    obs = rng.integers(-1, 12, size=(cap, N, T + 1, D)).astype(np.float32)
    act = rng.integers(0, A, size=(cap, N, T)).astype(np.int32)
    rew = (rng.random((cap, N, T)) < 0.2).astype(np.float32) * rng.random((cap, N, T)).astype(np.float32)
    if coop:
        rew[:] = rew[:, :1]
    length = rng.integers(1, T + 1, size=cap)
    done = np.zeros((cap, T + 1), np.uint8); filled = np.zeros((cap, T), np.uint8)
    for e in range(cap):
        filled[e, : length[e]] = 1
        done[e, length[e]] = rng.random() < 0.8
    return dict(obs=obs, act=act, rew=rew, done=done, filled=filled)


def ac_batch(rng, P, N, T, D, A=6, obs_high=8, coop=False):
    """An on-policy batch of P random episodes in the device layout (numpy arrays): ragged lengths, each ending in a terminal step, sparse
    rewards (`coop`: agent 0's reward for every agent)."""
    obs = rng.integers(-1, obs_high, size=(P, N, T + 1, D)).astype(np.float32)
    act = rng.integers(0, A, size=(P, N, T)).astype(np.int32)
    rew = (rng.random((P, N, T)) < 0.2).astype(np.float32) * rng.random((P, N, T)).astype(np.float32)
    if coop:
        rew[:] = rew[:, :1]
    length = rng.integers(1, T + 1, size=P)
    done = np.zeros((P, T + 1), np.uint8); filled = np.zeros((P, T), np.uint8)
    for e in range(P):
        filled[e, : length[e]] = 1
        done[e, length[e]] = 1
    return dict(obs=obs, act=act, rew=rew, done=done, filled=filled)


def traj_store(s, device):
    """a TrajStore holding the episodes of a device-layout batch / store (ac_batch, random_store)"""
    from codebase_b200.lbf import TrajStore

    cap, N, T1, D = s["obs"].shape
    ts = TrajStore(cap, N, T1 - 1, D, device)
    for k in ("obs", "act", "rew", "done", "filled"):
        getattr(ts, k).copy_(torch.as_tensor(s[k]))
    return ts


def ac_oracle_batch(s):
    """the device-layout batch in the layout of the reference's AC Batch: obss (T+1, P, N*D), actions / rewards (T, P, N), dones (T+1, P), filled (T, P)"""
    t = {k: torch.as_tensor(v) for k, v in s.items()}
    P, N, T1, D = t["obs"].shape
    return dict(obss=t["obs"].permute(2, 0, 1, 3).reshape(T1, P, N * D).float(), actions=t["act"].permute(2, 0, 1).long(),
                rewards=t["rew"].permute(2, 0, 1).float(), dones=t["done"].permute(1, 0).float(), filled=t["filled"].permute(1, 0).float())


def ac_model(hp, N, D, P, T, A=6, sharing=False, cls="A2CNetwork", centralised=False, standardise=False, num_epochs=4, ppo_clip=0.2):
    """an A2CNetwork / PPONetwork with the oracle's hyper-parameters (oracle.learner_ref.A2CHP): [128, 128] networks, orthogonal initialisation,
    room for P environments of T steps"""
    from codebase_b200.ac import model as M

    cfg = types.SimpleNamespace(optimizer="Adam", lr=hp.lr, gamma=hp.gamma, grad_clip=hp.grad_clip, n_steps=hp.n_steps, entropy_coef=hp.entropy_coef,
                                value_loss_coef=hp.value_loss_coef, target_update_interval_or_tau=hp.target_update_interval_or_tau,
                                standardise_returns=standardise, num_epochs=num_epochs, ppo_clip=ppo_clip)
    net = types.SimpleNamespace(layers=[128, 128], parameter_sharing=sharing, use_rnn=False, use_orthogonal_init=True, centralised=False)
    cnet = types.SimpleNamespace(**{**vars(net), "centralised": centralised})
    return getattr(M, cls)([space(shape=(D,))] * N, [space(n=A)] * N, cfg, net, cnet, "cuda", max_envs=P, max_episode_length=T)


def close_scaled(a, b, tol=1e-5):
    """element-wise, relative to the tensor's own scale (Adam's second moment lives at 1e-6 .. 1e-10).  For v = (1 - beta2) g^2 pass tol=2e-5:
    a relative gradient error e shows up as 2e in v, so 2e-5 on v is the 1e-5 bar on g."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    scale = max(float(np.abs(b).max()), 1e-30)
    assert np.abs(a - b).max() <= tol * scale, (float(np.abs(a - b).max()), scale)


def clipped(grad, max_norm):
    """clip_grad_norm_ on the host, from the device's normalised gradient: what the fused Adam step consumes"""
    if not max_norm:
        return grad
    norm = float(np.sqrt((grad.astype(np.float64) ** 2).sum()))
    return grad * min(1.0, max_norm / (norm + 1e-6))


TIE = 2e-5   # relative gap of the two best online Q-values under which the double-Q argmax may legitimately differ between two implementations


class NearTie(Exception):
    """The seeded case sits on a discontinuity of the loss gradient -- a double-Q argmax margin below TIE, a ReLU unit at its kink with a visible
    gradient share, a PPO ratio on the edge of the clip range -- or an oracle gradient too small to judge the element it updates: comparing
    against the oracle would be a coin toss.  The message says which."""


def check_margin(lr, st, batch, hp):
    margin = lr.double_q_margin(st, batch, hp)
    if margin < TIE:
        raise NearTie(f"double-Q argmax margin {margin:.1e}")


def assert_grad_close(lr, st, batch, hp, got, want, tol=1e-5, what="", kink_risk=None):
    """max |got - want| <= tol x max(1, max |want|).  A mismatch that a single ReLU unit sitting on its kink explains is a NearTie, not a failure: a
    hidden pre-activation within ~1e-6 of zero may be "on" in one implementation and "off" in the other (they agree to ~5e-7), which moves the
    gradient by up to dL/dh x (the unit's input row) = oracle.learner_ref.dqn_kink_risk -- e.g. 1.3e-3 for VDN at batch 16, T = 127, where the
    defect-free kernels of two consecutive builds "failed" this way.  The excuse only covers mismatches up to twice that bound.
    kink_risk: () -> that bound, for learners other than IDQN / VDN (QMIX: oracle.qmix_ref.qmix_kink_risk; A2C / PPO: a2c_kink_risk / ppo_kink_risk)."""
    import numpy as np

    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    scale = max(1.0, float(np.abs(want).max()))
    err = float(np.abs(got - want).max())
    if err <= tol * scale:
        return
    risk = kink_risk() if kink_risk is not None else lr.dqn_kink_risk(st, batch, hp)
    if risk >= 0.5 * err:
        raise NearTie(f"{what} ReLU kink: gradient error {err:.3e}, largest kink move {risk:.3e}")
    raise AssertionError(f"{what} max abs error {err:.3e} > {tol:g} x {scale:.3g} (largest ReLU-kink move of this case: {risk:.3e})")


def redraw_on_near_tie(fn):
    """Run the test body with seeds 0, 1, ... until it raises no NearTie (at most five draws): away from the loss gradient's discontinuities every
    mismatch is a defect; five near-ties in a row are not plausible (double-Q near-ties occur in ~8 % of random initialisations,
    tools/grad_stress.py).  Each re-draw is printed with its cause."""

    @functools.wraps(fn)
    def wrapper(*args, **kwargs):
        for attempt in range(5):
            torch.manual_seed(7919 * attempt + 17)
            try:
                return fn(*args, **kwargs)
            except NearTie as e:
                print(f"near-tie: {fn.__name__}{kwargs or args} re-drawn after initialisation {attempt}: {e}")   # shown by pytest -rP / -s
                continue
        pytest.fail("five initialisations in a row sat on a discontinuity of the loss gradient (near-tie): not plausible")

    return wrapper

"""GPU: IDQN, VDN, IA2C, IPPO, MAA2C and MAPPO from one to 32 agents (MARL_MAX_AGENTS) and 32 networks, against the oracle
(oracle/learner_ref.py, oracle/gru_ref.py, tests/gru_ac_ref.py) run in float64 from the learner's float32 parameters: one update per shape, the
forward passes, determinism, unglued update chains, update_n and the shapes the learners must refuse.

Everything that depends on the number of agents or networks -- make_plan's proportional CTA split, cta_rows / decode_row over up to 32 nets,
slot_agent for uneven parameter-sharing groups, the per-agent loss statistics, VDN's sum over agents, the per-agent td_ext stride of
standardise_returns, the centralised critic's joint input and the two-kernel optimiser tail -- runs at the shapes of real configurations
(Foraging-8x8-8p-2f: 8 agents x 30 features; Foraging-20x20-32p-10f: 32 x 126; RWARE large: 19 x 71).  H = 128 throughout.

  case                  learner          N   D    A  sharing            what it reaches
  idqn_n1_d30           IDQN             1   30   6  -                  tensor-core backward, one net; double-Q
  idqn_n8_d30           IDQN             8   30   6  independent        the 8p-2f shape: tensor-core forward and backward, 8 nets, in-kernel TD head
  vdn_n9_d30            VDN              9   30   6  independent        VDN's sum over 9 agents on the tensor-core path
  idqn_n16_d31_seps     IDQN             16  31   8  groups 13 / 2 / 1  widest tensor-core backward input (bias column 31), A = kOutPad, uneven split
  idqn_n32_d3           IDQN             32  3    6  independent        32 nets, one k-step
  vdn_n32_d32_shared    VDN              32  32   6  shared             tensor-core forward, FP32 training kernel (D = 32 has no spare column)
  idqn_n32_std          IDQN             32  12   6  independent        standardise_returns: 32 columns, per-agent td_ext into the tc backward
  idqn_rnn_n32          IDQN GRU         32  3    6  independent        GRU kernels over 32 nets
  vdn_rnn_n8            VDN GRU          8   30   6  independent        GRU kernels over 8 nets, VDN's sum
  ia2c_n32_d126         IA2C             32  126  6  independent        the 32p-10f shape: KP = 128, 32 actor and 32 critic nets
  ippo_n19_d71          IPPO             19  71   5  independent        the RWARE large shape, four epochs
  maa2c_n32_d4          MAA2C            32  4    6  shared actor       joint critic input exactly 128
  mappo_n8_d4           MAPPO            8   4    6  independent        joint input 32: critic and target critic on the tensor-core forward (row modes 2 / 3)
  maa2c_n6_d21          MAA2C            6   21   6  independent        the LBF 6p-1f shape, joint input 126
  ia2c_n32_std          IA2C             32  12   6  independent        standardise_returns at its 32-agent limit
  ia2c_rnn_n32          IA2C GRU         32  12   6  independent        GRU actor and critic kernels over 32 nets

Every per-network parameter block (W1, b1, ... of every net) of the first update's gradient must meet 1e-5 of that block's largest float64
magnitude (the critic's one-element output bias: of that sum without cancellation, _critic_bias_floors).  Later updates of a chain are
judged by the whole-vector bars of the existing chain tests: Adam's sign-led first steps on near-zero gradients move the two states apart there.  tests/test_agent_range.py checks, without a GPU, that each case still sits on the edge it claims.
"""
import copy
import ctypes as C
import dataclasses
import types

import numpy as np
import pytest
import torch

from oracle import gru_ref as gr
from oracle import learner_ref as lr
from oracle import policy_ref
from tests import gru_ac_ref as gar
from tests import test_rnn_ac_gpu as rac
from tests.helpers import NearTie, TIE, ac_batch, ac_oracle_batch, assert_grad_close, close_scaled, random_store, redraw_on_near_tie, space, traj_store

BLOCK_TOL = 1e-5         # gradient, per network and layer block, relative to the block's largest float64 element
SEED = 0x3200_A6E5
DQN = ("idqn", "vdn")
PPO = ("ippo", "mappo")
CENTRAL = ("maa2c", "mappo")


@dataclasses.dataclass(frozen=True)
class Case:
    kind: str                     # idqn, vdn, ia2c, ippo, maa2c, mappo
    N: int
    D: int
    A: int = 6
    sharing: object = False       # the actor's (DQN: the agents') parameter sharing: False, True or a tuple of group labels
    critic_sharing: object = False
    rnn: bool = False             # GRU agents (DQN) / GRU actor (actor-critic)
    critic_rnn: object = None     # GRU critic (None: as rnn)
    H: int = 128                  # hidden width of the agents (DQN) / the actor
    critic_H: int = 128
    B: int = 16                   # DQN: episodes per batch; actor-critic: environments (n_envs)
    T: int = 8
    double_q: bool = False
    standardise: bool = False
    tu: float = 3.0               # target_update_interval_or_tau
    epochs: int = 2               # PPO

    @property
    def dqn(self):
        return self.kind in DQN

    @property
    def joint(self):
        """the critic's input width (a centralised critic reads all N observations side by side)"""
        return self.N * self.D if self.kind in CENTRAL and self.N > 1 else self.D

    @property
    def crnn(self):
        return self.rnn if self.critic_rnn is None else self.critic_rnn

    @property
    def tc_backward(self):
        """the DQN family's three-kernel tensor-core training pass takes MLP agents with D < 32 (column D carries the bias)"""
        return self.dqn and not self.rnn and self.D < 32


SEPS = (0, 1, 0, 0, 2, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0)   # 13 / 2 / 1 agents, the groups interleaved

CASES = {
    "idqn_n1_d30": Case("idqn", 1, 30, double_q=True, B=16, T=8),
    "idqn_n8_d30": Case("idqn", 8, 30, B=16, T=10),
    "vdn_n9_d30": Case("vdn", 9, 30, B=12, T=8),
    "idqn_n16_d31_seps": Case("idqn", 16, 31, A=8, sharing=SEPS, B=12, T=8),
    "idqn_n32_d3": Case("idqn", 32, 3, B=16, T=8),
    "vdn_n32_d32_shared": Case("vdn", 32, 32, sharing=True, B=8, T=6, tu=0.05),
    "idqn_n32_std": Case("idqn", 32, 12, standardise=True, B=12, T=8),
    "idqn_rnn_n32": Case("idqn", 32, 3, rnn=True, B=8, T=6),
    "vdn_rnn_n8": Case("vdn", 8, 30, rnn=True, B=12, T=8),
    "ia2c_n32_d126": Case("ia2c", 32, 126, B=8, T=6, tu=2.0),
    "ippo_n19_d71": Case("ippo", 19, 71, A=5, B=12, T=8, epochs=4),
    "maa2c_n32_d4": Case("maa2c", 32, 4, sharing=True, B=8, T=6),
    "mappo_n8_d4": Case("mappo", 8, 4, B=16, T=10, tu=2.0),
    "maa2c_n6_d21": Case("maa2c", 6, 21, B=16, T=8),
    "ia2c_n32_std": Case("ia2c", 32, 12, standardise=True, B=8, T=6),
    "ia2c_rnn_n32": Case("ia2c", 32, 12, rnn=True, B=8, T=6),
}


def _opt(name, on):
    from codebase_b200 import _native as nat

    nat.check(nat.lib().marl_set_option(name, C.c_int32(int(on))), "marl_set_option")


@pytest.fixture(autouse=True)
def _restore():
    yield
    _opt(b"tensor_core_backward", True)   # the library defaults
    _opt(b"tensor_core_forward", True)


def _sharing(s):
    return list(s) if isinstance(s, tuple) else s


def _f64(batch):
    return {k: v.double() if v.is_floating_point() else v for k, v in batch.items()}


def _ret_ms64(shape):
    ms = lr.RunningMeanStdRef(shape)
    ms.mean, ms.var = ms.mean.double(), ms.var.double()
    return ms


def _blocks(m):
    """(name, slice) of every layer block of every network in the flat parameter vector ([actor | critic] for the actor-critic learners)"""
    parts = [("net", m.n_nets, m._shapes)] if hasattr(m, "_shapes") else [("actor", m.n_actor_nets, m._actor_shapes), ("critic", m.n_critic_nets, m._critic_shapes)]
    out, o = [], 0
    for part, n_nets, shapes in parts:
        for k in range(n_nets):
            for name, shape in shapes:
                size = int(np.prod(shape))
                out.append((f"{part}{k}.{name}", slice(o, o + size)))
                o += size
    return out


def _assert_blocks(m, got, want, what, kink_risk, other=None, floors=None):
    """every layer block within BLOCK_TOL x its largest float64 element (with `other`: got against other on the same scale).  A miss that a
    ReLU unit on its kink explains is a NearTie, as in tests.helpers.assert_grad_close.  floors: {block: scale}, a lower bound of a block's scale
    (_critic_bias_floors).  Returns (worst block, its fraction of the bar)."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    ref = want if other is None else np.asarray(other, np.float64)
    ratios, errs = {}, {}
    for name, sl in _blocks(m):
        errs[name] = float(np.abs(got[sl] - ref[sl]).max())
        ratios[name] = errs[name] / (BLOCK_TOL * max(float(np.abs(want[sl]).max()), (floors or {}).get(name, 0.0), 1e-30))
    bad = {k: round(v, 2) for k, v in ratios.items() if not v <= 1.0}
    if bad:
        err = max(errs[k] for k in bad)
        risk = kink_risk()
        if risk >= 0.5 * err:
            raise NearTie(f"{what}: ReLU kink: block error {err:.3e}, largest kink move {risk:.3e}")
        worst = sorted(bad, key=bad.get)[-8:]
        raise AssertionError(f"{what}: {len(bad)} gradient blocks over {BLOCK_TOL:g} x their largest element (fraction of the bar): "
                             f"{ {k: bad[k] for k in worst} } (largest ReLU-kink move {risk:.3e})")
    worst = max(ratios, key=ratios.get)
    return worst, ratios[worst]


# ---- the DQN family ------------------------------------------------------------------------------------------------------------------------------
def _dqn_hp(c):
    return lr.DqnHP(grad_clip=1.0, double_q=c.double_q, target_update_interval_or_tau=c.tu, mixer=1 if c.kind == "vdn" else 0)


def _dqn_model(c):
    from codebase_b200.dqn import model as M

    hp = _dqn_hp(c)
    cfg = types.SimpleNamespace(optimizer="Adam", lr=hp.lr, gamma=hp.gamma, grad_clip=hp.grad_clip, double_q=c.double_q, target_update_interval_or_tau=c.tu,
                                standardise_returns=c.standardise)
    cls = M.VDNetwork if c.kind == "vdn" else M.QNetwork
    return cls([space(shape=(c.D,))] * c.N, [space(n=c.A)] * c.N, cfg, [c.H, c.H], _sharing(c.sharing), c.rnn, True, "cuda", max_batch=c.B, max_episode_length=c.T)


def _dqn_perturb(m):
    """a target that differs from the online networks, so that the target pass matters"""
    m.theta_tgt.copy_(m.theta + 0.01 * torch.randn_like(m.theta))
    m.params_changed()


def _dqn_copy(dst, src):
    dst.theta.copy_(src.theta); dst.theta_tgt.copy_(src.theta_tgt)
    dst.params_changed()


def _dqn_oracle(c, m):
    f = lambda t: t.detach().cpu().double().clone()   # noqa: E731
    ret_ms = _ret_ms64((1,) if c.kind == "vdn" else (c.N,)) if c.standardise else None
    return lr.DqnState(f(m.theta), f(m.theta_tgt), list(m.agent_net), c.D, c.A, ret_ms=ret_ms)


def _dqn_store(c, seed, cap=None):
    s = random_store(np.random.default_rng(seed), cap or c.B, c.N, c.T, c.D, c.kind == "vdn", A=c.A)
    if c.rnn:   # LBF-like magnitudes keep the GRU away from saturation
        s["obs"] = (s["obs"] / 6.0).astype(np.float32)
    return s


def _dqn_ref(c):
    """the oracle module of the case's agents: MLP (learner_ref) or GRU (gru_ref; tests/gru_ac_ref.py at a width below 128)"""
    return (gr if c.H == gr.H else gar) if c.rnn else lr


def _dqn_margin(c, st, b, hp):
    if c.double_q:
        margin = _dqn_ref(c).double_q_margin(st, b, hp)
        if margin < TIE:
            raise NearTie(f"double-Q argmax margin {margin:.1e}")


def _dqn_step(c, m, st, b64, hp, ts, idx):
    """one update on the device and in the oracle: (state before, oracle result, device metrics)"""
    _dqn_margin(c, st, b64, hp)
    st0 = copy.deepcopy(st)
    want = _dqn_ref(c).dqn_update(st, b64, hp)
    met = m.update_from_store(ts, idx).cpu().numpy()
    return st0, want, met


def _check_dqn(c, m, st, st0, b64, want, met, hp, what, u=0, per_block=True):
    """loss, filled count, the gradient (per block, or the whole-vector bar), clip norm, Adam m / v, parameters and target, running statistics"""
    n = m.n_params
    g = m.grad.cpu().numpy().astype(np.float64)
    fill = float(b64["filled"].sum())
    assert g[n + 1] == fill and met[4] == fill, (what, g[n + 1], met[4], fill)
    assert abs(float(met[0]) - want["loss"]) <= 1e-5 * max(1.0, abs(want["loss"])), f"loss, {what}: {float(met[0])} vs {want['loss']}"
    kink = lambda: _dqn_ref(c).dqn_kink_risk(st0, b64, hp)   # noqa: E731
    got = g[:n] / fill
    worst = None
    if per_block:
        worst = _assert_blocks(m, got, want["grad"].numpy(), what, kink)
    else:
        assert_grad_close(lr, st0, b64, hp, got, want["grad"].numpy(), tol=1e-5, what=what, kink_risk=kink)
    assert abs(float(met[1]) - want["grad_norm"]) <= 1e-5 * max(1.0, want["grad_norm"]), f"clip norm, {what}: {float(met[1])} vs {want['grad_norm']}"
    mtol = 5e-5 if c.rnn else 2e-5 if c.standardise else 1e-5   # the Adam bars of test_rnn_dqn_gpu.py / test_update_chain_gpu.py
    close_scaled(m.adam_m.cpu().numpy(), st.m.numpy(), mtol); close_scaled(m.adam_v.cpu().numpy(), st.v.numpy(), 2 * mtol)
    for name, mine, theirs in (("theta", m.theta, st.theta), ("target", m.theta_tgt, st.theta_tgt)):
        d = np.abs(mine.cpu().numpy().astype(np.float64) - theirs.numpy())
        assert np.quantile(d, 0.999) < 1e-5 and d.max() < 2 * hp.lr * (u + 1) + 1e-6, (what, name, float(np.quantile(d, 0.999)), float(d.max()))
    if c.standardise:
        mean, var, count = m.ret_ms()
        for got_ms, ref in ((mean, st.ret_ms.mean), (var, st.ret_ms.var)):
            np.testing.assert_allclose(got_ms.numpy(), ref.numpy().reshape(-1), rtol=1e-5, atol=1e-5, err_msg=what)
        assert abs(count - st.ret_ms.count) < 1e-6 * count, (what, count, st.ret_ms.count)
    return worst


# ---- the actor-critic learners: the per-update checks of tests/test_rnn_ac_gpu.py (MLP or GRU parts) ---------------------------------------------
def _rcase(c):
    """the case in tests/test_rnn_ac_gpu.py's terms, for its per-update checks"""
    return rac.Case(ppo=c.kind in PPO, arnn=c.rnn, crnn=c.crnn, N=c.N, D=c.D, A=c.A, sharing=c.sharing, centralised=c.kind in CENTRAL, P=c.B, T=c.T,
                    tu=c.tu, grad_clip=0.5, epochs=c.epochs, standardise=c.standardise)


def _ac_model(c, epochs=None):
    from codebase_b200.ac import model as M

    hp = rac._hp(_rcase(c))
    cfg = types.SimpleNamespace(optimizer="Adam", lr=hp.lr, gamma=hp.gamma, grad_clip=hp.grad_clip, n_steps=hp.n_steps, entropy_coef=hp.entropy_coef,
                                value_loss_coef=hp.value_loss_coef, target_update_interval_or_tau=hp.target_update_interval_or_tau,
                                standardise_returns=c.standardise, num_epochs=epochs or c.epochs, ppo_clip=0.2)
    anet = types.SimpleNamespace(layers=[c.H, c.H], parameter_sharing=_sharing(c.sharing), use_rnn=c.rnn, use_orthogonal_init=True, centralised=False)
    cnet = types.SimpleNamespace(layers=[c.critic_H, c.critic_H], parameter_sharing=_sharing(c.critic_sharing), use_rnn=c.crnn, use_orthogonal_init=True,
                                 centralised=c.kind in CENTRAL)
    cls = M.PPONetwork if c.kind in PPO else M.A2CNetwork
    return cls([space(shape=(c.D,))] * c.N, [space(n=c.A)] * c.N, cfg, anet, cnet, "cuda", max_envs=c.B, max_episode_length=c.T)


def _ac_oracle(c, m):
    f = lambda t: t.detach().cpu().double().clone()   # noqa: E731
    return lr.A2CState(f(m.theta[: m.n_actor]), f(m.theta[m.n_actor:]), f(m.theta_tgt), list(m.actor_net), list(m.critic_net), c.D, c.A,
                       centralised=c.kind in CENTRAL, ret_ms=_ret_ms64((c.N,)) if c.standardise else None)


def _ac_batch(c, seed):
    s = ac_batch(np.random.default_rng(seed), c.B, c.N, c.T, c.D, A=c.A)
    if c.rnn or c.crnn:
        s["obs"] = (s["obs"] / 6.0).astype(np.float32)
    return s


def _critic_bias_floors(m, st0, b64, hp, returns):
    """The critic's output bias is one element whose gradient is a plain sum over its agents' filled rows of 2 x value_loss_coef x (V - R) /
    filled: where those terms cancel, the sum is far smaller than the terms a float32 reduction rounds.  Its scale is the same sum without the
    cancellation, 2 x value_loss_coef x sum |R - V| / filled (R: the returns the loss reads, V: the critic before the update), in float64."""
    obs = list(torch.split(b64["obss"], st0.in_dim, dim=-1))
    cobs, CD = st0.critic_inputs(obs)
    with torch.no_grad():
        v = torch.cat(gar.agents_forward(st0.critic, st0.critic_net, [o[:-1] for o in cobs], CD, 1), dim=-1)   # (T, P, N)
    per_agent = ((returns - v).abs() * b64["filled"].unsqueeze(-1)).sum((0, 1)) * 2 * hp.value_loss_coef / b64["filled"].sum()
    bias = m._critic_shapes[-1][0]
    return {f"critic{k}.{bias}": float(sum(per_agent[a] for a, n in enumerate(st0.critic_net) if n == k)) for k in set(st0.critic_net)}


def _ac_step(c, m, st, s, hp, step, tr, what, per_block):
    """one update of the device and the oracle, then every per-update check of test_rnn_ac_gpu.py; per_block: the gradient per block too (PPO:
    the first epoch's, from a second handle stopped after one epoch).  Returns the worst block."""
    b64 = _f64(ac_oracle_batch(s))
    st0 = copy.deepcopy(st)
    want = rac._oracle_update(_rcase(c), st, b64, hp, step)
    return _ac_check(c, m, st, st0, b64, want, traj_store(s, m.device), hp, step, tr, what, per_block)


def _ac_check(c, m, st, st0, b64, want, ts, hp, step, tr, what, per_block, floors=None):
    """_ac_step's device update and checks against an oracle update already taken (st0: the oracle's state before it, st: after, want: its
    result), so that several handles can be held to one oracle update; ts: the store, whose first c.B environments are the batch b64; floors:
    more blocks' scales for _assert_blocks"""
    rc = _rcase(c)
    th0, tgt0 = m.theta.detach().clone(), m.theta_tgt.detach().clone()
    met = m.update_from_store(ts, c.B, step).cpu().numpy()
    worst = None
    if per_block:
        fill = float(b64["filled"].sum())
        n = m.n_actor + m.n_critic
        if c.kind in PPO:
            m1 = _ac_model(c, epochs=1)
            m1.theta.copy_(th0); m1.theta_tgt.copy_(tgt0)
            m1.update_from_store(ts, c.B, step)
            got, ref = m1.grad.cpu().numpy()[:n] / fill, want["grads"][0]
            kink = lambda: gar.ppo_kink_risk(st0, b64, hp, want, 0.2, 0)   # noqa: E731
            m1.close()
        else:
            got, ref = m.grad.cpu().numpy()[:n] / fill, want["grad"]
            kink = lambda: gar.a2c_kink_risk(st0, b64, hp)   # noqa: E731
        worst = _assert_blocks(m, got, np.concatenate([ref["actor"].numpy(), ref["critic"].numpy()]), what, kink,
                               floors={**_critic_bias_floors(m, st0, b64, hp, want["returns"]), **(floors or {})})
    rac._check_update(m, rc, hp, st, st0, b64, want, met, step, tgt0.cpu().numpy(), tr, what)
    return worst


# ---- 1. one update per case against the float64 oracle ------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", [k for k, c in CASES.items() if c.dqn])
@redraw_on_near_tie
def test_dqn_update_matches_the_float64_oracle(name):
    """ragged episodes through marl_dqn_update: loss, gradient per block, clip norm, Adam state, parameters and target, running statistics.  A
    case the tensor-core backward takes runs with tensor_core_backward 1 and 0 on two handles of the same parameters: each meets the oracle, and
    their gradients agree per block on the same bar"""
    c = CASES[name]
    hp = _dqn_hp(c)
    forms = (1, 0) if c.tc_backward else (None,)
    models = [_dqn_model(c) for _ in forms]
    _dqn_perturb(models[0])
    for m in models[1:]:
        _dqn_copy(m, models[0])
    st = _dqn_oracle(c, models[0])
    s = _dqn_store(c, int(torch.randint(0, 1 << 30, (1,))))
    b64 = _f64(lr.batch_from_store(s, np.arange(c.B)))
    ts = traj_store(s, models[0].device)
    idx = torch.arange(c.B, dtype=torch.int32, device=models[0].device)
    _dqn_margin(c, st, b64, hp)
    st0 = copy.deepcopy(st)
    want = _dqn_ref(c).dqn_update(st, b64, hp)
    grads = []
    for form, m in zip(forms, models):
        if form is not None:
            _opt(b"tensor_core_backward", form)
        met = m.update_from_store(ts, idx).cpu().numpy()
        what = f"{name}" + ("" if form is None else f", tensor_core_backward={form}")
        blk, ratio = _check_dqn(c, m, st, st0, b64, want, met, hp, what)
        print(f"{what}: worst gradient block {blk} at {ratio:.3f} of the {BLOCK_TOL:g} bar")
        grads.append(m.grad.cpu().numpy()[: m.n_params].astype(np.float64) / float(b64["filled"].sum()))
    if len(grads) == 2:
        blk, ratio = _assert_blocks(models[0], grads[0], want["grad"].numpy(), f"{name}: tensor-core vs FP32 backward",
                                    lambda: _dqn_ref(c).dqn_kink_risk(st0, b64, hp), other=grads[1])
        print(f"{name}: tensor-core vs FP32 backward, worst block {blk} at {ratio:.3f} of the bar")
    for m in models:
        m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", [k for k, c in CASES.items() if not c.dqn])
@redraw_on_near_tie
def test_ac_update_matches_the_float64_oracle(name):
    """one update (hard sync or Polyak step at step 0): gradient per block, then returns, target values, advantages, raw and clipped gradient,
    loss / entropy / value metrics, grad norm, Adam m / v per block, parameters, target critic, running statistics"""
    c = CASES[name]
    m = _ac_model(c)
    rac._perturb_target(m)
    st = _ac_oracle(c, m)
    hp = rac._hp(_rcase(c))
    s = _ac_batch(c, int(torch.randint(0, 1 << 30, (1,))))
    blk, ratio = _ac_step(c, m, st, s, hp, 0, rac.Tracker(m.n_actor + m.n_critic), name, per_block=True)
    print(f"{name}: worst gradient block {blk} at {ratio:.3f} of the {BLOCK_TOL:g} bar")
    m.close()


# ---- 2. forward passes -------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("N,D,E", [(32, 3, 20000), (8, 30, 4096)])
def test_q_values_tensor_core_and_ffma_match_the_oracle(N, D, E):
    """q_values of online and target networks: the tensor-core forward and the FFMA forward each against the float64 oracle and against each
    other, to 1e-5 of the largest |Q|"""
    torch.manual_seed(N * D)
    c = Case("idqn", N, D, B=4, T=2)
    m = _dqn_model(c)
    _dqn_perturb(m)
    obs = torch.randint(-1, 12, (E, N, D)).float()
    xs = [obs[:, a].double() for a in range(N)]
    for target, flat in ((False, m.theta), (True, m.theta_tgt)):
        want = torch.stack(lr.agents_forward(flat.cpu().double(), list(m.agent_net), xs, D, c.A), 1).numpy()
        got = {}
        for tc in (1, 0):
            _opt(b"tensor_core_forward", tc)
            got[tc] = m.q_values(obs.cuda(), target=target).cpu().numpy().astype(np.float64)
        scale = max(1.0, float(np.abs(want).max()))
        for what, a, b in (("tensor-core", got[1], want), ("FFMA", got[0], want), ("tensor-core vs FFMA", got[1], got[0])):
            err = float(np.abs(a - b).max())
            assert err <= 1e-5 * scale, f"{what} q_values (target={target}): max error {err:.3e}, scale {scale:.3g}"
    m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["mappo_n8_d4", "maa2c_n32_d4"])
def test_logits_and_values_match_the_oracle(name):
    """logits, values and values(target=True) with the centralised critic at joint widths 32 and 128"""
    c = CASES[name]
    torch.manual_seed(c.N)
    m = _ac_model(c)
    rac._perturb_target(m)
    E = 1000
    obs = torch.randint(-1, 8, (E, c.N, c.D)).float()
    xs = [obs[:, a].double() for a in range(c.N)]
    joint = [obs.reshape(E, c.N * c.D).double()] * c.N
    for got, flat, nets, inputs, ind, out in ((m.logits(obs.cuda()), m.theta[: m.n_actor], m.actor_net, xs, c.D, c.A),
                                              (m.values(obs.cuda()), m.theta[m.n_actor:], m.critic_net, joint, c.joint, 1),
                                              (m.values(obs.cuda(), target=True), m.theta_tgt, m.critic_net, joint, c.joint, 1)):
        want = torch.stack(lr.agents_forward(flat.cpu().double(), list(nets), inputs, ind, out), 1).reshape(got.shape)
        np.testing.assert_allclose(got.cpu().numpy(), want.numpy(), rtol=1e-5, atol=1e-5 * max(1.0, float(want.abs().max())))
    m.close()


# ---- 3. determinism at N = 32 ------------------------------------------------------------------------------------------------------------------
def _state(m):
    out = dict(theta=m.theta, theta_tgt=m.theta_tgt, adam_m=m.adam_m, adam_v=m.adam_v, grad=m.grad, metrics=m._metrics)
    out = {k: v.detach().cpu().clone() for k, v in out.items()}
    if m.standardise_returns:
        mean, var, count = m.ret_ms()
        out.update(ret_mean=mean, ret_var=var, ret_count=torch.tensor(count, dtype=torch.float64))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", [k for k, c in CASES.items() if c.N == 32])
def test_second_handle_repeats_the_update_bit_for_bit(name):
    c = CASES[name]
    torch.manual_seed(32)
    if c.dqn:
        a, b = _dqn_model(c), _dqn_model(c)
        _dqn_perturb(a); _dqn_copy(b, a)
        ts = traj_store(_dqn_store(c, 5), a.device)
        idx = torch.arange(c.B, dtype=torch.int32, device=a.device)
        for m in (a, b):
            m.update_from_store(ts, idx)
    else:
        a, b = _ac_model(c), _ac_model(c)
        rac._perturb_target(a)
        b.theta.copy_(a.theta); b.theta_tgt.copy_(a.theta_tgt)
        ts = traj_store(_ac_batch(c, 5), a.device)
        for m in (a, b):
            m.update_from_store(ts, c.B, 0)
    got, want = _state(a), _state(b)
    for k in want:
        assert torch.equal(got[k], want[k]), f"{k}: max abs difference {float((got[k].double() - want[k].double()).abs().max()):.3e}"
    a.close(); b.close()


# ---- 4. unglued three-update chains --------------------------------------------------------------------------------------------------------------
CHAINS = {
    "idqn_n8_d30_hard": dataclasses.replace(CASES["idqn_n8_d30"], tu=2.0),            # hard sync of the target at update 2
    "vdn_n32_d32_shared_polyak": CASES["vdn_n32_d32_shared"],                          # Polyak target every update
    "ia2c_n32_d126": CASES["ia2c_n32_d126"],                                           # hard syncs at steps 0 and 4
    "mappo_n8_d4": CASES["mappo_n8_d4"],                                               # odd steps: the perturbed target critic is never synced
}
# environment step of each actor-critic update (hard syncs where step % tu == 0)
AC_STEPS = {"ia2c_n32_d126": (0, 3, 4), "mappo_n8_d4": (1, 3, 5)}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CHAINS))
@redraw_on_near_tie
def test_unglued_chain_matches_the_float64_oracle(name):
    """three updates, the device and the oracle never re-synchronised; the first update is judged per block, later ones by the chain tests' bars"""
    c = CHAINS[name]
    if c.dqn:
        hp = _dqn_hp(c)
        m = _dqn_model(c)
        _dqn_perturb(m)
        st = _dqn_oracle(c, m)
        idx = torch.arange(c.B, dtype=torch.int32, device=m.device)
        for u in range(3):
            s = _dqn_store(c, 1000 * u + int(torch.randint(0, 1 << 20, (1,))))
            b64 = _f64(lr.batch_from_store(s, np.arange(c.B)))
            st0, want, met = _dqn_step(c, m, st, b64, hp, traj_store(s, m.device), idx)
            _check_dqn(c, m, st, st0, b64, want, met, hp, f"{name}, update {u}", u=u, per_block=u == 0)
        assert m.updates == 3
        if c.tu > 1:
            assert st.last_target_update == 2
    else:
        m = _ac_model(c)
        rac._perturb_target(m)
        st = _ac_oracle(c, m)
        hp = rac._hp(_rcase(c))
        tr = rac.Tracker(m.n_actor + m.n_critic)
        seed = int(torch.randint(0, 1 << 20, (1,)))
        for u, step in enumerate(AC_STEPS[name]):
            _ac_step(c, m, st, _ac_batch(c, seed + u), hp, step, tr, f"{name}, update {u}", per_block=u == 0)
    m.close()


# ---- 5. update_n at N = 8 and 32: the loop it replaces, on the two-kernel optimiser tail -----------------------------------------------------------
UPDATE_N = {"idqn_n8_d30": CASES["idqn_n8_d30"], "idqn_n32_d3": CASES["idqn_n32_d3"]}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(UPDATE_N))
def test_update_n_is_the_loop_it_replaces(name):
    """8 x 21254 and 32 x 17798 parameters exceed the fused reduce + Adam tail's one wave (132 x 512): both run grad_reduce_kernel + adam_kernel"""
    from codebase_b200 import _native as nat

    c, K, cap = UPDATE_N[name], 4, 48
    torch.manual_seed(c.N)
    a, b = _dqn_model(c), _dqn_model(c)
    _dqn_perturb(a); _dqn_copy(b, a)
    ts = traj_store(_dqn_store(c, c.N * 100 + c.B, cap), a.device)
    a.update_n(ts, c.B, cap, SEED, 0, K)
    idx = torch.zeros(c.B, dtype=torch.int32, device=b.device)
    for u in range(K):
        nat.check(nat.lib().marl_replay_sample(C.c_uint64(SEED), C.c_uint64(u), C.c_int32(c.B), C.c_int32(cap), nat.ptr(idx), nat.stream_ptr()), "marl_replay_sample")
        assert np.array_equal(idx.cpu().numpy(), policy_ref.replay_sample(SEED, u, c.B, cap)), f"replay indices of update {u}"
        b.update_from_store(ts, idx)
    got, want = _state(a), _state(b)
    for k in want:
        assert torch.equal(got[k], want[k]), f"{k}: max abs difference {float((got[k].double() - want[k].double()).abs().max()):.3e}"
    assert a.updates == b.updates == K
    a.close(); b.close()


# ---- 6. the acceptance edges ---------------------------------------------------------------------------------------------------------------------
KINDS = ("idqn", "vdn", "ia2c", "ippo", "maa2c", "mappo")


def _model(c):
    return _dqn_model(c) if c.dqn else _ac_model(c)


def _train_once(m, c):
    """one update on random episodes: finite metrics, every parameter finite, the parameters moved"""
    theta0 = m.theta.clone()
    if c.dqn:
        met = m.update_from_store(traj_store(_dqn_store(c, 9), m.device), torch.arange(c.B, dtype=torch.int32, device=m.device)).cpu().numpy()
    else:
        met = m.update_from_store(traj_store(_ac_batch(c, 9), m.device), c.B, 0).cpu().numpy()
    assert np.isfinite(met).all() and met[4] > 0, met
    assert bool(torch.isfinite(m.theta).all()) and float((m.theta - theta0).abs().max()) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_every_learner_is_created_and_trains_at_32_agents(kind):
    c = Case(kind, 32, 4, B=8, T=6)
    m = _model(c)
    assert m.n_agents == 32 and (m.n_nets if c.dqn else m.n_critic_nets) == 32
    _train_once(m, c)
    m.close()


def _native_create(which, n_agents, critic_in=None):
    from codebase_b200 import _native as nat

    lib, h = nat.lib(), C.c_void_p()
    nets = (C.c_int32 * nat.MAX_AGENTS)(*range(min(n_agents, nat.MAX_AGENTS)))
    cfg = nat.MlpCfg(n_agents, min(n_agents, nat.MAX_AGENTS), nets, 4, 128, 6)
    if which == "dqn":
        hp = nat.DqnHP(3e-4, 0.99, 1.0, 1, 200.0, 0.9, 0.999, 1e-8, 0)
        nat.check(lib.marl_dqn_create(C.byref(cfg), C.byref(hp), C.c_int32(8), C.c_int32(6), C.c_int32(0), C.byref(h)), "marl_dqn_create")
    else:
        ccfg = nat.MlpCfg(n_agents, min(n_agents, nat.MAX_AGENTS), nets, critic_in or 4, 128, 1)
        hp = nat.A2cHP(3e-4, 0.99, 0.5, 5, 0.001, 0.5, 200.0, 0.9, 0.999, 1e-8)
        nat.check(lib.marl_a2c_create(C.byref(cfg), C.byref(ccfg), C.byref(hp), C.c_int32(8), C.c_int32(6), C.c_int32(0), C.byref(h)), "marl_a2c_create")
    return h


REFUSED = {**{f"{k}_n33": k for k in KINDS}, "dqn_create_n33": "native", "a2c_create_n33": "native", "maa2c_n32_d5_joint160": "joint",
           "a2c_create_critic160": "native"}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(REFUSED))
def test_refused_shapes_fail_cleanly_and_leave_the_device_usable(name):
    """33 agents raise NotImplementedError in every learner before any native call; marl_dqn_create / marl_a2c_create refuse n_agents = 33 with
    MARL_EINVAL; a centralised critic of 32 x 5 = 160 inputs is refused in Python and by marl_a2c_create.  After each refusal the device has no
    pending error and a learner created next trains."""
    from codebase_b200 import _native as nat

    why = REFUSED[name]
    if why in KINDS:
        with pytest.raises(NotImplementedError, match=r"33 agents: the learners take at most 32 agents"):
            _model(Case(why, 33, 3))
    elif why == "joint":
        with pytest.raises(NotImplementedError, match=r"joint observation is 32 x 5 = 160 wide"):
            _model(Case("maa2c", 32, 5))
    elif name == "dqn_create_n33":
        with pytest.raises(nat.NativeError, match=r"marl_dqn_create failed \(rc=-1\): marl_dqn_create: n_agents out of range"):
            _native_create("dqn", 33)
    elif name == "a2c_create_n33":
        with pytest.raises(nat.NativeError, match=r"marl_a2c_create failed \(rc=-1\): marl_a2c_create\(actor\): n_agents out of range"):
            _native_create("a2c", 33)
    else:
        with pytest.raises(nat.NativeError, match=r"marl_a2c_create failed \(rc=-1\): marl_a2c_create\(critic\): obs dim 160 not supported \(1\.\.128\)"):
            _native_create("a2c", 32, critic_in=160)
    torch.cuda.synchronize()
    c = Case("idqn" if name.startswith(("idqn", "vdn", "dqn")) else "mappo", 32, 4, B=8, T=6)
    m = _model(c)
    _train_once(m, c)
    m.close()


# ---- 7. the drivers end to end -------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("alg,env,N,extra", [
    ("idqn", "Foraging-8x8-8p-2f-v3", 8, ["algorithm.batch_size=32", "algorithm.buffer_size=512", "algorithm.updates_per_iteration=4"]),
    ("ia2c", "Foraging-20x20-32p-10f-v3", 32, []),
])
def test_driver_trains_at_many_agents(alg, env, N, extra, tmp_path, monkeypatch):
    import pandas as pd

    from codebase_b200 import run

    monkeypatch.chdir(tmp_path)
    run.main([f"+algorithm={alg}", f"env.name=lbforaging:{env}", "env.time_limit=25", "env.parallel_envs=64", "seed=0", "algorithm.total_steps=8000",
              "algorithm.eval_interval=2000", f"run_dir={tmp_path}/out", *extra])
    df = pd.read_csv(tmp_path / "out" / "results.csv")
    for k in range(N):
        assert f"agent{k}/mean_episode_returns" in df.columns, df.columns.tolist()
    losses = [col for col in df.columns if "loss" in col]
    assert losses and len(df) >= 2 and all(np.isfinite(df[col].iloc[-1]) for col in losses), df[losses].tail()

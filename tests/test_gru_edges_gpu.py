"""GPU: the recurrent (GRU) kernels (csrc/gru_kernels.cu) at every class of their sequence split, at hidden widths 1-128, inputs 1-128 and 1-8
actions, at T = 1, 2 and 100, in the act step, on a reused handle and at the loss head's block edges, against the float64 oracle.

gru_backward_kernel walks each CTA's run of sequences in 16-sequence tiles of two 8-sequence halves (tests/row_plan.py explains the 12 classes and
the three net-level cases).  The split follows the device's SM count, so every case reads it from the device and picks its batch with
row_plan.find_units: a GPU with another SM count still runs every class.  The episode of the first and the last sequence of every CTA and of every
tile (row_plan.cta_edge_sequences) is filled at every step, so losing or doubling such a sequence moves the gradient: tests/test_gru_edges.py
shows, without a GPU, that it moves some block past the bar on 114 and 132 SMs.

Every case is one update from perturbed parameters (online != target), compared with the float64 oracle (oracle/gru_ref.py and
tests/gru_ac_ref.py; tests/hidden_width_ref.py's networks below H = 128): every layer block of every network within 1e-5 of its largest float64
element (test_agent_range_gpu._assert_blocks), then the loss, the filled count, Adam's m / v, the parameters and the target (DQN family:
test_agent_range_gpu._check_dqn; actor-critic: test_rnn_ac_gpu._check_update through test_agent_range_gpu._ac_step, PPO's first epoch per block).
At every multi-tile class a second handle given the same inputs repeats the gradient bit for bit."""
import copy
import dataclasses

import numpy as np
import pytest
import torch

from oracle import gru_ref as gr
from oracle import learner_ref as lr
from oracle import qmix_ref as qr
from tests import gru_ac_ref as gar
from tests import row_plan as rp
from tests import test_agent_range_gpu as ar
from tests import test_rnn_ac_gpu as rac
from tests import test_rnn_dqn_gpu as rdq
from tests.helpers import ac_oracle_batch, redraw_on_near_tie, traj_store

MAX_SEQS = 7_000           # sequences N B per case: the float64 oracle stays quick
SEPS = ar.SEPS             # 16 agents in groups of 13 / 2 / 1, interleaved
GROUPS4 = (0, 1, 0, 0)     # 4 agents in groups of 3 / 1
DQN = ("idqn", "vdn", "qmix")
PPO = ("ippo", "mappo")
CENTRAL = ("maa2c", "mappo")


@dataclasses.dataclass(frozen=True)
class Case:
    kind: str                  # idqn, vdn, qmix, ia2c, ippo, maa2c, mappo
    N: int
    D: int
    A: int = 6
    sharing: object = False    # the agents' / the actor's and the critic's parameter sharing: False, True or a tuple of group labels
    T: int = 4
    H: int = 128               # hidden width of the agents / the actor
    critic_H: int = 128
    arnn: bool = True          # actor-critic: recurrent actor
    crnn: bool = True          # actor-critic: recurrent critic
    cls: str = None            # the class the case runs at (None: its key in CLASS_CASES)

    @property
    def dqn(self):
        return self.kind in DQN

    def part(self):
        """(in_dim, out_dim) of the recurrent part whose split the case's class names: the agents, else the actor, else the critic"""
        if self.dqn or self.arnn:
            return self.D, self.A
        return (self.N * self.D if self.kind in CENTRAL and self.N > 1 else self.D), 1


CLASS_CASES = {
    "t1-lower": Case("idqn", 2, 9, T=6),
    "t1-half": Case("vdn", 4, 12, sharing=True, T=5),
    "t1-upper": Case("ia2c", 16, 7, sharing=SEPS, T=6),
    "t1-full": Case("ippo", 4, 10, sharing=GROUPS4, T=5),
    "t2-lower": Case("maa2c", 2, 8, sharing=True, T=3),
    "t2-half": Case("mappo", 2, 6, T=3),
    "t2-upper": Case("idqn", 4, 11, sharing=GROUPS4, T=3),
    "t2-full": Case("ia2c", 2, 15, crnn=False, T=2),
    "t3+-lower": Case("vdn", 2, 10, T=2),
    "t3+-half": Case("ippo", 2, 9, sharing=True, T=2),
    "t3+-upper": Case("maa2c", 2, 5, arnn=False, T=2),
    "t3+-full": Case("idqn", 1, 13, A=4, T=2),
    rp.GRU_SMALL_NET: Case("qmix", 3, 9, T=8),
    rp.GRU_ONE_CTA: Case("mappo", 2, 12, sharing=True, T=8),
    rp.GRU_STRADDLE: Case("ia2c", 5, 9, sharing=True, A=5, T=3),   # 5 agents: agent boundaries fall inside CTAs on 114 and 132 SMs
}

# hidden widths 1, 2, 37, 100, 127 (actor and critic of different widths); inputs 1, 31, 32 (DQN: the last KX = 32 template and the first
# width it takes) and 33, 64, 128 (actor-critic: KX = 128), a joint critic input of exactly 128 (N = 4, D = 32); every action count 1, 2, 3, 5, 8
WIDTH_CASES = {
    "idqn_h1_d1_a1": Case("idqn", 2, 1, A=1, H=1, cls="t2-upper"),
    "vdn_h37_d31_a3": Case("vdn", 2, 31, A=3, H=37, cls="t3+-lower", T=2),
    "idqn_h127_d32_a8": Case("idqn", 3, 32, A=8, H=127, sharing=True, cls="t2-upper", T=2),
    "ia2c_h2_d33_a2_c100": Case("ia2c", 2, 33, A=2, H=2, critic_H=100, cls="t2-upper", T=2),
    "ippo_h100_d64_a5_c37": Case("ippo", 2, 64, A=5, H=100, critic_H=37, sharing=True, cls="t3+-lower", T=2),
    "ia2c_h127_d128_a3_c2": Case("ia2c", 2, 128, A=3, H=127, critic_H=2, cls="t2-upper", T=2),
    "maa2c_h37_joint128_a8_c127": Case("maa2c", 4, 32, A=8, H=37, critic_H=127, sharing=GROUPS4, cls="t2-upper", T=2),
}

# episode length: T = 1 (W_hh gets no gradient from the zero state), T = 2, and long BPTT (T = 100) at a t1 class
LENGTH_CASES = {
    "idqn_T1": Case("idqn", 2, 9, T=1, cls="t2-upper"),
    "ia2c_T1": Case("ia2c", 2, 9, T=1, cls="t2-lower"),
    "vdn_T2": Case("vdn", 2, 7, T=2, cls="t2-half"),
    "idqn_T100": Case("idqn", 2, 9, T=100, cls="t1-upper"),
    "vdn_T100": Case("vdn", 2, 6, T=100, sharing=True, cls="t1-lower"),
    "ippo_T100": Case("ippo", 2, 8, T=100, cls="t1-upper"),
}

# act step: sharing groups, H = 37 and 128, at E = 1, 17 and 9001 environments
ACT_CASES = {
    "idqn_h37_groups": Case("idqn", 3, 11, sharing=(0, 0, 1), H=37),
    "vdn_h128_shared": Case("vdn", 2, 15, sharing=True),
    "mappo_h128_c37": Case("mappo", 2, 13, critic_H=37),
    "ia2c_h37_c128_groups": Case("ia2c", 4, 9, sharing=GROUPS4, H=37),
}
ACT_E = (1, 17, 9001)

# handle reuse: created at (2 B, 2 T), trained at (B, T) of a multi-tile class
REUSE_CASES = {"idqn": Case("idqn", 2, 9, T=3, cls="t2-upper"), "ia2c": Case("ia2c", 2, 9, T=3, cls="t2-lower")}

# the loss head reduces per 256 rows of N P T: exactly 2 blocks (N = 2, P = 64, T = 4), one row more (N = 3, P = 57, T = 3), below one block
HEAD_CASES = {"ia2c_npt512": (Case("ia2c", 2, 9, T=4), 64), "ippo_npt513": (Case("ippo", 3, 9, T=3, sharing=True), 57),
              "mappo_npt30": (Case("mappo", 2, 9, T=3), 5)}


def all_train_cases():
    """every training case of the file: (name, case) with its class"""
    out = [(k, dataclasses.replace(c, cls=k)) for k, c in CLASS_CASES.items()]
    return out + list(WIDTH_CASES.items()) + list(LENGTH_CASES.items()) + list(REUSE_CASES.items())


def n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def units(c, sm):
    """B (sequences per agent) of the case on sm SMs; a class out of reach fails (a device with another SM count must not quietly test less)"""
    B = rp.find_units(c.N, c.sharing, sm, c.cls, MAX_SEQS)
    assert B is not None, f"{c.cls}: no batch of {c} within {MAX_SEQS} sequences reaches it on {sm} SMs"
    return B


def acase(c, B, T=None):
    """the case in test_agent_range_gpu's terms (max_batch / max_envs B, max_episode_length T)"""
    return ar.Case(c.kind, c.N, c.D, A=c.A, sharing=c.sharing, critic_sharing=c.sharing, rnn=c.dqn or c.arnn, critic_rnn=None if c.dqn else c.crnn,
                   B=B, T=c.T if T is None else T, H=c.H, critic_H=c.critic_H, epochs=2)


def data(c, B, sm, seed):
    """seeded episodes in the device layout (DQN: a replay store of B episodes; actor-critic: B environments); the episode of every edge sequence
    of the plan on sm SMs is filled at every step"""
    ac = acase(c, B)
    s = ar._dqn_store(ac, seed) if c.dqn else ar._ac_batch(ac, seed)
    if c.kind == "qmix":
        s["rew"][:] = s["rew"][:, :1]
    full = sorted({b for _, b in rp.cta_edge_sequences(rp.gru_plan(rp.nets_of(c.N, c.sharing), B, sm))})
    s["filled"][full] = 1; s["done"][full] = 0; s["done"][full, c.T] = 1
    return s, full


def dqn_hp(c):
    return lr.DqnHP(grad_clip=1.0, double_q=False, target_update_interval_or_tau=3.0, mixer={"vdn": 1, "qmix": 2}.get(c.kind, 0))


def qmix_state(c, theta, theta_tgt, mix, mix_tgt):
    return qr.QmixState(theta, theta_tgt, mix, mix_tgt, rp.nets_of(c.N, c.sharing), c.D, c.A, rdq.MIXING["embed_dim"], rdq.MIXING["hypernet_embed"])


# ---- one update on the device against the oracle ------------------------------------------------------------------------------------------------
def _qmix_model(c, B, T):
    qc = rdq.Case(mixer=2, N=c.N, D=c.D, A=c.A, sharing=list(c.sharing) if isinstance(c.sharing, tuple) else c.sharing, B=B, T=T, double_q=False, cap=B)
    return rdq._learner(qc)


def _train_qmix(c, B, what, seed, twin):
    """QMIX (H = 128): update_grads, the agents' gradient per block and the mixer's to 1e-5 of its largest element, the loss and filled count"""
    m = _qmix_model(c, B, c.T)
    m.theta_tgt.copy_(m.theta + 0.02 * torch.randn_like(m.theta)); m.params_changed()
    f = lambda t: t.detach().cpu().double().clone()   # noqa: E731
    st = qmix_state(c, f(m.theta), f(m.theta_tgt), f(m.mix), f(m.mix_tgt))
    s, full = data(c, B, n_sm(), seed)
    b64 = ar._f64(lr.batch_from_store(s, np.arange(B)))
    hp = dqn_hp(c)
    st0 = copy.deepcopy(st)
    want = gr.qmix_update(st, b64, hp)
    ts = traj_store(s, m.device)
    idx = torch.arange(B, dtype=torch.int32, device=m.device)
    m.update_grads(ts, idx)
    g = m.grad.cpu().numpy().astype(np.float64)
    n, fill = m.n_params, float(b64["filled"].sum())
    assert g[n + 1] == fill, (what, g[n + 1], fill)
    assert abs(g[n] / fill - want["loss"]) <= 1e-5 * max(1.0, abs(want["loss"])), (what, g[n] / fill, want["loss"])
    worst = ar._assert_blocks(m, g[:n] / fill, want["grad"].numpy(), what, lambda: gr.qmix_kink_risk(st0, b64, hp))
    mg, wm = m.mix_grad[: m.n_mix].cpu().numpy().astype(np.float64) / fill, want["mix_grad"].numpy()
    assert np.abs(mg - wm).max() <= 1e-5 * np.abs(wm).max(), (what, "mixer gradient", float(np.abs(mg - wm).max()), float(np.abs(wm).max()))
    if twin:
        m2 = _qmix_model(c, B, c.T)
        for k in ("theta", "theta_tgt", "mix", "mix_tgt"):
            getattr(m2, k).copy_(getattr(m, k))
        m2.params_changed()
        m2.update_grads(ts, idx)
        assert torch.equal(m.grad, m2.grad) and torch.equal(m.mix_grad, m2.mix_grad), f"{what}: a second handle differs"
        m2.close()
    m.close()
    return worst, full


def _twin_equal(a, b, what):
    for k in ("grad", "theta", "theta_tgt", "adam_m", "adam_v"):
        x, y = getattr(a, k), getattr(b, k)
        assert torch.equal(x, y), f"{what}: {k} of a second handle differs (max abs difference {float((x.double() - y.double()).abs().max()):.3e})"


def train(c, B, what, seed, twin=False, make=None, warm=None):
    """one update of the case at B (sequences per agent) against the oracle; twin: a second handle of the same parameters repeats it bit for
    bit; make: the (B, T) the handle is created at (handle reuse; the twin is then created at the case's own shape); warm: a batch the handle
    trains on first, its parameters reset after.  Returns (worst block, its fraction of the bar, the edge episodes)."""
    if c.kind == "qmix":
        (blk, ratio), full = _train_qmix(c, B, what, seed, twin)
        return blk, ratio, full
    ac = acase(c, *(make or (B, c.T)))
    m = ar._dqn_model(ac) if c.dqn else ar._ac_model(ac)
    (ar._dqn_perturb if c.dqn else rac._perturb_target)(m)
    m2 = None
    if twin:
        m2 = ar._dqn_model(acase(c, B)) if c.dqn else ar._ac_model(acase(c, B))
        m2.theta.copy_(m.theta); m2.theta_tgt.copy_(m.theta_tgt)
        if c.dqn:
            m2.params_changed()
    if warm is not None:
        th, tg = m.theta.clone(), m.theta_tgt.clone()
        if c.dqn:
            m.update_grads(traj_store(warm, m.device), torch.arange(warm["obs"].shape[0], dtype=torch.int32, device=m.device))
        else:
            m.update_grads(traj_store(warm, m.device), warm["obs"].shape[0])
        assert bool(torch.isfinite(m.grad).all()), what
        m.theta.copy_(th); m.theta_tgt.copy_(tg)
        if c.dqn:
            m.params_changed()
    s, full = data(c, B, n_sm(), seed)
    assert all(bool(s["filled"][b].all()) for b in full), what   # every edge sequence carries gradient at every step
    ac = acase(c, B)
    ts = traj_store(s, m.device)
    if c.dqn:
        hp = ar._dqn_hp(ac)
        st = ar._dqn_oracle(ac, m)
        b64 = ar._f64(lr.batch_from_store(s, np.arange(B)))
        idx = torch.arange(B, dtype=torch.int32, device=m.device)
        st0, want, met = ar._dqn_step(ac, m, st, b64, hp, ts, idx)
        blk, ratio = ar._check_dqn(ac, m, st, st0, b64, want, met, hp, what)
        if m2 is not None:
            m2.update_from_store(ts, idx)
    else:
        st = ar._ac_oracle(ac, m)
        hp = rac._hp(ar._rcase(ac))
        blk, ratio = ar._ac_step(ac, m, st, s, hp, 0, rac.Tracker(m.n_actor + m.n_critic), what, per_block=True)
        if m2 is not None:
            m2.update_from_store(ts, B, 0)
    if m2 is not None:
        _twin_equal(m, m2, what)
        m2.close()
    if c.T == 1:   # the zero initial state gives W_hh nothing: exactly 0.0 on the device, as in the oracle
        zero = [sl for name, sl in ar._blocks(m) if name.endswith("rnn.weight_hh_l0")]
        assert zero and all(not m.grad[sl].any() for sl in zero), f"{what}: a W_hh gradient element is not 0.0 at T = 1"
    m.close()
    return blk, ratio, full


def _report(name, c, B, blk, ratio, full):
    sm = n_sm()
    print(f"{sm} SMs: {name}: class {c.cls} ({c.kind}, N={c.N}, sharing={c.sharing}, D={c.D}, A={c.A}, H={c.H}/{c.critic_H}, B={B}, T={c.T}, "
          f"{c.N * B} sequences, {len(full)} edge episodes): worst block {blk} at {ratio:.3f} of the {ar.BLOCK_TOL:g} bar")


# ---- 1. one case per class ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_the_class_sweep_covers_every_class_on_this_device():
    sm = n_sm()
    covered = set()
    for cls, c in CLASS_CASES.items():
        covered |= rp.gru_classes(tuple(rp.nets_of(c.N, c.sharing)), units(dataclasses.replace(c, cls=cls), sm), sm)
    print(f"{sm} SMs: the class sweep covers {sorted(covered)}")
    assert covered >= set(rp.GRU_CLASSES), sorted(set(rp.GRU_CLASSES) - covered)


@pytest.mark.gpu
@pytest.mark.parametrize("cls", list(CLASS_CASES))
@redraw_on_near_tie
def test_class_matches_the_float64_oracle(cls):
    c = dataclasses.replace(CLASS_CASES[cls], cls=cls)
    B = units(c, n_sm())
    multi = cls.startswith(("t2", "t3")) or cls == rp.GRU_STRADDLE
    blk, ratio, full = train(c, B, f"{cls} ({c.kind}, N={c.N}, B={B}, T={c.T})", int(torch.randint(0, 1 << 30, (1,))), twin=multi)
    _report(cls, c, B, blk, ratio, full)


# ---- 2. widths and action counts -----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(WIDTH_CASES))
@redraw_on_near_tie
def test_width_matches_the_float64_oracle(name):
    c = WIDTH_CASES[name]
    B = units(c, n_sm())
    blk, ratio, full = train(c, B, f"{name} ({c.cls}, B={B})", int(torch.randint(0, 1 << 30, (1,))), twin=True)
    _report(name, c, B, blk, ratio, full)


# ---- 3. episode length -------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(LENGTH_CASES))
@redraw_on_near_tie
def test_episode_length_matches_the_float64_oracle(name):
    c = LENGTH_CASES[name]
    B = units(c, n_sm())
    blk, ratio, full = train(c, B, f"{name} ({c.cls}, B={B})", int(torch.randint(0, 1 << 30, (1,))), twin=c.cls.startswith(("t2", "t3")))
    _report(name, c, B, blk, ratio, full)


# ---- 4. the act step ---------------------------------------------------------------------------------------------------------------------------
def _close(got, want, what):
    want = want.numpy()
    err = float(np.abs(got.cpu().numpy().astype(np.float64) - want).max())
    assert err <= 1e-5 * max(1.0, float(np.abs(want).max())), f"{what}: max error {err:.3e}"


@pytest.mark.gpu
@pytest.mark.parametrize("E", ACT_E)
@pytest.mark.parametrize("name", list(ACT_CASES))
def test_act_steps_carry_h_like_the_oracle(name, E):
    """three carried steps of marl_dqn_forward_rnn / marl_a2c_forward_rnn (actor, critic, target critic): outputs and the compact [E][N][H] h
    against tests/hidden_width_ref.act_steps at every step"""
    c = ACT_CASES[name]
    torch.manual_seed(E + c.N)
    S = 3
    obs = (torch.randint(-1, 12, (S, E, c.N, c.D)) / 6.0).float()
    ac = acase(c, 4, 2)
    if c.dqn:
        m = ar._dqn_model(ac)
        ar._dqn_perturb(m)
        parts = [("q", lambda o, h: m.q_values(o, h=h), m.theta, m.agent_net, obs, c.D, c.A, c.H),
                 ("target q", lambda o, h: m.q_values(o, target=True, h=h), m.theta_tgt, m.agent_net, obs, c.D, c.A, c.H)]
    else:
        m = ar._ac_model(ac)
        rac._perturb_target(m)
        cobs = gar.joint(obs) if c.kind in CENTRAL else obs
        parts = [("logits", lambda o, h: m.logits(o, h=h), m.theta[: m.n_actor], m.actor_net, obs, c.D, c.A, c.H),
                 ("values", lambda o, h: m.values(o, h=h), m.theta[m.n_actor:], m.critic_net, cobs, m.critic_in, 1, c.critic_H),
                 ("target values", lambda o, h: m.values(o, target=True, h=h), m.theta_tgt, m.critic_net, cobs, m.critic_in, 1, c.critic_H)]
    for what, fwd, flat, nets, x, ind, outd, H in parts:
        want_o, want_h = gar.act_steps(flat.detach().cpu().double(), list(nets), x.double(), ind, outd)
        h = None
        for s in range(S):
            out, h_new = fwd(obs[s].cuda().contiguous(), h)
            assert tuple(h_new.shape) == (E, c.N, H), (what, tuple(h_new.shape))
            _close(out.reshape(want_o[s].shape), want_o[s], f"{name}, E={E}: {what} step {s}")
            _close(h_new, want_h[s], f"{name}, E={E}: {what} h step {s}")
            h = h_new.clone()
    m.close()


# ---- 5. a handle reused below the shape it was created for ---------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(REUSE_CASES))
@redraw_on_near_tie
def test_handle_reused_at_a_smaller_batch_matches_a_fresh_one(name):
    """a handle created at (2 B, 2 T) trains first on a (2 B, 2 T) batch of 1e3-scaled observations, then, parameters reset, on (B, T) of a
    multi-tile class: the oracle's checks hold and a fresh handle created at (B, T) repeats it bit for bit (row_index and the gru_save pitch
    follow the call, not the handle)"""
    c = REUSE_CASES[name]
    B = units(c, n_sm())
    seed = int(torch.randint(0, 1 << 30, (1,)))
    big = dataclasses.replace(c, T=2 * c.T)
    warm, _ = data(big, 2 * B, n_sm(), seed + 1)
    warm["obs"] = (warm["obs"] * 1e3).astype(np.float32)
    blk, ratio, full = train(c, B, f"reused {name} handle ({c.cls}, B={B})", seed, twin=True, make=(2 * B, 2 * c.T), warm=warm)
    _report(f"reused {name}", c, B, blk, ratio, full)


# ---- 6. the loss head's statistics blocks ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(HEAD_CASES))
@redraw_on_near_tie
def test_head_blocks_match_the_float64_oracle(name):
    """gru_ac_head_kernel's four metrics over N P T = 512, 513 and 30 rows (test_rnn_ac_gpu._check_update), the gradient per block"""
    c, P = HEAD_CASES[name]
    assert (c.N * P * c.T) % 256 in (0, 1) or c.N * P * c.T < 256
    ac = acase(c, P)
    m = ar._ac_model(ac)
    rac._perturb_target(m)
    st = ar._ac_oracle(ac, m)
    s = ar._ac_batch(ac, int(torch.randint(0, 1 << 30, (1,))))
    blk, ratio = ar._ac_step(ac, m, st, s, rac._hp(ar._rcase(ac)), 0, rac.Tracker(m.n_actor + m.n_critic), name, per_block=True)
    print(f"{name}: N P T = {c.N * P * c.T}: worst block {blk} at {ratio:.3f} of the bar")
    m.close()


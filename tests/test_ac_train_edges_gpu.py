"""GPU: the actor-critic MLP training pass (learner_kernels.cu: train_kernel<KP, kHeadA2cCritic> and <KP, kHeadA2cActor>, a2c.cu's
a2c_gradients) at every branch class of its row split, at KP = 16, 32, 64 and 128, hidden widths 1-128, 1-8 actions and joint critic inputs up
to 128, and the forward kernels (mlp_forward_kernel, tc_forward_kernel) of the act step at every class of the dense split, against the float64
oracle.

Each pass of an update walks the rows of episode_plan over its own networks (tests/row_plan.py explains the 24 classes and the two small-net
cases): the critic pass over cplan, writing each row's advantage, the actor pass over aplan, reading it.  The two plans differ where the critic's
parameter sharing differs from the actor's.  The split follows the device's SM count, so every case reads it from the device and picks its
batch with row_plan.find_batch: a GPU with another SM count still runs every class.  The episode that ends a CTA of either pass has its full
length T, so every CTA's tail rows carry a loss; the other episodes are ragged.  tests/test_ac_train_edges.py shows, without a GPU, that losing
or doubling one such row moves some gradient block past the bar on 114 and 132 SMs.

Every training case is one update from perturbed parameters (no bias is zero, the target critic differs from the critic), held to the oracle
by test_agent_range_gpu's checks: every layer block of the gradient within 1e-5 of its largest float64 element (PPO: the first epoch's, per
block; the output biases of the actor and the critic on the scale of their sums without cancellation), then returns, target values and
advantages of every row t < T, losses, entropy, filled count, grad norm, Adam m / v, θ and the target critic (PPO: after all epochs).  Where the
target-critic or the old-log-prob pass can run on the tensor cores (128-wide networks, an input of at most 32), the update runs once with
tensor_core_forward on and once off, each against the oracle.  At every multi-tile class a second handle repeats the update bit for bit."""
import copy
import dataclasses

import numpy as np
import pytest
import torch

from oracle import learner_ref as lr
from tests import gru_ac_ref as gar
from tests import row_plan as rp
from tests import test_agent_range_gpu as ar
from tests import test_rnn_ac_gpu as rac
from tests.helpers import ac_oracle_batch, redraw_on_near_tie, traj_store

MAX_ROWS = 20_000                # rows N P (T + 1) per case: the float64 oracle stays quick
TS_ALL = tuple(range(8, 400))    # up to 3+ tiles of one episode per CTA
TS_SHORT = tuple(range(4, 64))   # several episodes per CTA
TS_MANY = tuple(range(20, 64))   # a few hundred episodes: several per CTA at a multi-tile class, tile boundaries inside an episode
SEPS = ar.SEPS                   # 16 agents in groups of 13 / 2 / 1, interleaved
GROUPS4 = (0, 1, 0, 0)           # 4 agents in groups of 3 / 1
GROUPS3 = (0, 1, 0)              # 3 agents in groups of 2 / 1
PPO = ("ippo", "mappo")
CENTRAL = ("maa2c", "mappo")
MAX_OBS_TC = 32                  # kMaxObsDim: the tensor-core forward's widest input
SAME = "same"                    # critic_sharing: as the actor's


@dataclasses.dataclass(frozen=True)
class Case:
    kind: str                    # ia2c, ippo, maa2c, mappo
    N: int
    D: int
    A: int = 6
    sharing: object = False      # the actor's parameter sharing: False, True or a tuple of group labels
    critic_sharing: object = SAME
    T_choices: tuple = TS_ALL
    H: int = 128                 # the actor's hidden width
    critic_H: int = 128
    standardise: bool = False
    epochs: int = 2              # PPO
    cls: str = None              # the class the case runs at (None: its key in CLASS_CASES)

    @property
    def csharing(self):
        return self.sharing if self.critic_sharing == SAME else self.critic_sharing

    @property
    def joint(self):
        """the critic's input width (a centralised critic reads all N observations side by side)"""
        return self.N * self.D if self.kind in CENTRAL and self.N > 1 else self.D

    @property
    def tc_forward(self):
        """a forward pass of the update can run on the tensor cores: the target critic's (critic input <= 32) or PPO's old log-probs' (actor
        input <= 32), with both networks 128 wide (no tensor-core image otherwise)"""
        return self.H == self.critic_H == 128 and (self.joint <= MAX_OBS_TC or (self.kind in PPO and self.D <= MAX_OBS_TC))


CLASS_CASES = {
    "t1-c1-full": Case("ippo", 2, 12, sharing=True, T_choices=TS_SHORT),
    "t1-c1-part": Case("maa2c", 3, 11),                              # joint 33: critic KP 64
    "t1-c2-full": Case("ia2c", 1, 40, A=8),
    "t1-c2-part": Case("mappo", 4, 8, sharing=GROUPS4, epochs=3),
    "t1-c3-full": Case("ia2c", 2, 17, standardise=True),
    "t1-c3-part": Case("ia2c", 16, 10, sharing=SEPS),
    "t1-c4-full": Case("ippo", 4, 100, sharing=True),
    "t1-c4-part": Case("maa2c", 3, 20, sharing=GROUPS3, critic_sharing=True),
    "t2-c1-full": Case("ia2c", 1, 128),
    "t2-c1-part": Case("mappo", 2, 33, sharing=True),                # joint 66
    "t2-c2-full": Case("ia2c", 4, 16, sharing=GROUPS4, critic_sharing=True),
    "t2-c2-part": Case("ippo", 3, 65, T_choices=TS_MANY),
    "t2-c3-full": Case("maa2c", 2, 64),                              # joint 128
    "t2-c3-part": Case("ia2c", 4, 20, sharing=True, T_choices=TS_MANY),
    "t2-c4-full": Case("ippo", 1, 32, epochs=4),
    "t2-c4-part": Case("mappo", 8, 16),                              # actor KP 16, critic KP 128
    "t3+-c1-full": Case("ia2c", 2, 1, A=2, sharing=True),
    "t3+-c1-part": Case("ippo", 1, 31, epochs=3),
    "t3+-c2-full": Case("maa2c", 3, 9),                              # joint 27: the target pass on the tensor cores
    "t3+-c2-part": Case("ia2c", 4, 45, sharing=GROUPS4, critic_sharing=False, standardise=True),
    "t3+-c3-full": Case("mappo", 2, 64),
    "t3+-c3-part": Case("ia2c", 1, 100, A=5),
    "t3+-c4-full": Case("ippo", 4, 20, sharing=True),
    "t3+-c4-part": Case("maa2c", 2, 8),                              # joint 16
    rp.SMALL_NET: Case("ippo", 2, 7, T_choices=TS_SHORT),
    rp.ONE_CTA: Case("mappo", 3, 11, sharing=True),
}

# inputs 1, 16, 17, 32, 33, 64, 65, 127, 128 (the KP = 16 / 32 / 64 / 128 tile edges); hidden widths 1, 2, 37, 100, 127 with actor and critic of
# different widths; every action count 1, 2, 3, 5, 8; joint critic inputs 32, 33, 64, 65, 128.  Each at a multi-tile class with a partial last tile.
WIDTH_CASES = {
    "ia2c_d1_a1_h1_c37": Case("ia2c", 2, 1, A=1, H=1, critic_H=37, cls="t2-c1-part"),
    "ippo_d16_a2_h2_c100": Case("ippo", 1, 16, A=2, H=2, critic_H=100, cls="t3+-c2-part"),
    "ia2c_d17_a3_h37_c127": Case("ia2c", 2, 17, A=3, H=37, critic_H=127, cls="t2-c3-part"),
    "mappo_joint32_a5_h100_c2": Case("mappo", 2, 16, A=5, H=100, critic_H=2, cls="t3+-c4-part"),
    "maa2c_joint33_a8_h127_c1": Case("maa2c", 3, 11, A=8, H=127, critic_H=1, cls="t2-c2-part"),
    "ia2c_d32_a8_c100": Case("ia2c", 1, 32, A=8, critic_H=100, cls="t3+-c1-part"),
    "ippo_d33_a1_h37": Case("ippo", 2, 33, A=1, H=37, cls="t2-c4-part"),
    "maa2c_joint64_a2_h2_c127": Case("maa2c", 2, 32, A=2, H=2, critic_H=127, cls="t3+-c3-part"),
    "ia2c_d64_a5_h100_c1": Case("ia2c", 1, 64, A=5, H=100, critic_H=1, cls="t2-c1-part"),
    "mappo_joint65_a3_h127_c37": Case("mappo", 5, 13, A=3, H=127, critic_H=37, cls="t3+-c2-part"),
    "ippo_d65_a8_h1_c2": Case("ippo", 2, 65, A=8, H=1, critic_H=2, cls="t2-c3-part"),
    "ia2c_d127_a2_h127_c100": Case("ia2c", 1, 127, A=2, H=127, critic_H=100, cls="t3+-c4-part"),
    "maa2c_joint128_a5_h37_c100": Case("maa2c", 2, 64, A=5, H=37, critic_H=100, cls="t2-c1-part"),
    "ia2c_d128_a3_h2_c37": Case("ia2c", 2, 128, A=3, H=2, critic_H=37, cls="t3+-c1-part"),
}

# T = 1 and 2 at multi-tile classes; one environment of T = 383 (384 rows: one episode over three tiles of one CTA)
LENGTH_CASES = {
    "ia2c_T1": Case("ia2c", 2, 9, T_choices=(1,), cls="t2-c1-part"),
    "ippo_T1": Case("ippo", 1, 12, T_choices=(1,), epochs=1, cls="t2-c1-part"),   # one epoch: ratio 1, no clip edge
    "mappo_T2": Case("mappo", 2, 7, T_choices=(2,), cls="t2-c1-part"),
    "ia2c_T383": Case("ia2c", 1, 20, T_choices=(383,), cls="t3+-c4-full"),
    "ippo_T383": Case("ippo", 2, 40, T_choices=(383,), cls="t3+-c4-full"),
}

# handle reuse: created at (2 P, 2 T), trained at (P, T) of a t2 and a t3+ class from a store of capacity 2 P
REUSE_CASES = {
    "ia2c_t2": Case("ia2c", 2, 20, cls="t2-c3-part"),
    "ippo_t3": Case("ippo", 2, 12, sharing=True, cls="t3+-c1-part"),
}


def all_train_cases():
    """every training case of the file: (name, case) with its class"""
    out = [(k, dataclasses.replace(c, cls=k)) for k, c in CLASS_CASES.items()]
    return out + list(WIDTH_CASES.items()) + list(LENGTH_CASES.items()) + list(REUSE_CASES.items())


def n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(autouse=True)
def _restore():
    yield
    ar._opt(b"tensor_core_forward", True)   # the library default


def shape(c, sm):
    """(P, T) of the case on sm SMs; a class out of reach fails (a device with another SM count must not quietly test less)"""
    found = rp.find_batch(c.N, c.sharing, c.T_choices, sm, c.cls, MAX_ROWS)
    assert found is not None, f"{c.cls}: no batch of {c} within {MAX_ROWS} rows reaches it on {sm} SMs"
    return found


def acase(c, P, T):
    """the case in test_agent_range_gpu's terms (n_envs P, episode length T)"""
    return ar.Case(c.kind, c.N, c.D, A=c.A, sharing=c.sharing, critic_sharing=c.csharing, H=c.H, critic_H=c.critic_H, B=P, T=T,
                   standardise=c.standardise, tu=3.0, epochs=c.epochs)


def edge_episodes(c, P, T, sm):
    """the episodes that end a CTA of the critic pass or of the actor pass on sm SMs"""
    return sorted(set(rp.last_episodes(rp.nets_of(c.N, c.sharing), P, T, sm)) | set(rp.last_episodes(rp.nets_of(c.N, c.csharing), P, T, sm)))


def data(c, P, T, sm, seed, cap=None):
    """seeded ragged episodes of P environments (a store of `cap` >= P, the first P the batch); the edge episodes run their full length T"""
    s = ar._ac_batch(acase(c, cap or P, T), seed)
    full = edge_episodes(c, P, T, sm)
    s["filled"][full] = 1; s["done"][full] = 0; s["done"][full, T] = 1
    return s, full


def perturb(m):
    """parameters off the initialisation: every bias non-zero, so that a row of zero observations still reaches every layer and carries a
    loss, and a target critic apart from the critic"""
    m.theta.add_(0.01 * torch.randn_like(m.theta))
    rac._perturb_target(m)


def actor_bias_floors(c, m, st0, b64, hp, want):
    """The actor's output bias gets the plain sum over its agents' filled rows of dL/dlogits.  Softmax's gradient sums to 0 over the actions (at
    two actions the two elements are one sum and its negation), and rows of either sign cancel: the sum can be far smaller than the terms a
    float32 reduction rounds, as for the critic's bias (test_agent_range_gpu._critic_bias_floors).  Its scale is the same sum of |dL/dlogit|
    (PPO: the first epoch's surrogate), in float64."""
    actor, critic = st0.actor.clone().requires_grad_(True), st0.critic.clone()
    logits = []

    def forward(flat, agent_net, xs, in_dim, out_dim):
        out = gar.agents_forward(flat, agent_net, xs, in_dim, out_dim)
        if flat is actor:
            for y in out:
                y.retain_grad()
            logits.extend(out)
        return out

    saved, lr.agents_forward = lr.agents_forward, forward
    try:
        if c.kind in PPO:
            loss = lr.ppo_losses(actor, critic, st0, b64, hp, want["returns"], want["old_logp"], 0.2)[1]
        else:
            loss = lr.a2c_losses(actor, critic, st0.target, copy.deepcopy(st0), b64, hp)[0]
        loss.backward()
    finally:
        lr.agents_forward = saved
    per_agent = [y.grad.abs().sum((0, 1)) for y in logits]   # (A,) per agent
    bias = m._actor_shapes[-1][0]
    return {f"actor{k}.{bias}": float(sum(g for a, g in enumerate(per_agent) if st0.actor_net[a] == k).max()) for k in set(st0.actor_net)}


def _batch64(s, P):
    return ar._f64(ac_oracle_batch({k: v[:P] for k, v in s.items()}))


def _states_equal(a, b, what):
    for k in ("grad", "theta", "theta_tgt", "adam_m", "adam_v", "_metrics"):
        x, y = getattr(a, k), getattr(b, k)
        assert torch.equal(x, y), f"{what}: {k} differs (max abs difference {float((x.double() - y.double()).abs().max()):.3e})"


def train(c, P, T, what, seed, twin=False, make=None, warm=None, cap=None):
    """one update of the case at (P, T) against the oracle, with tensor_core_forward on and off where a forward pass can take the tensor cores;
    twin: a second handle of the same parameters repeats it bit for bit; make: the (P, T) the handle is created at (the twin is created at the
    case's own); warm: a store whose gradients the handle takes first (no optimiser step); cap: the store's capacity.  Returns the worst block and
    its fraction of the bar over the forms."""
    ac = acase(c, P, T)
    forms = (1, 0) if c.tc_forward else (None,)
    models = [ar._ac_model(acase(c, *make) if make else ac) for _ in forms]
    perturb(models[0])
    twins = [ar._ac_model(ac)] if twin else []
    for m in models[1:] + twins:
        m.theta.copy_(models[0].theta); m.theta_tgt.copy_(models[0].theta_tgt)
    if warm is not None:   # gradients only: the optimiser's state stays that of a fresh handle
        for m in models:
            tw = traj_store(warm, m.device)
            if c.kind in PPO:
                m.epoch_grads(tw, warm["obs"].shape[0], 0)
            else:
                m.update_grads(tw, warm["obs"].shape[0])
            assert bool(torch.isfinite(m.grad).all()), what
    s, full = data(c, P, T, n_sm(), seed, cap)
    b64 = _batch64(s, P)
    assert all(bool(b64["filled"][:, b].all()) for b in full), what
    ts = traj_store(s, models[0].device)
    st = ar._ac_oracle(ac, models[0])
    hp = rac._hp(ar._rcase(ac))
    st0 = copy.deepcopy(st)
    want = rac._oracle_update(ar._rcase(ac), st, b64, hp, 0)
    floors = actor_bias_floors(c, models[0], st0, b64, hp, want)
    worst = ("", 0.0)
    for form, m in zip(forms, models):
        if form is not None:
            ar._opt(b"tensor_core_forward", form)
        w = what + ("" if form is None else f", tensor_core_forward={form}")
        blk, ratio = ar._ac_check(ac, m, copy.deepcopy(st), st0, b64, want, ts, hp, 0, rac.Tracker(m.n_actor + m.n_critic), w, per_block=True,
                                   floors=floors)
        worst = max(worst, (blk, ratio), key=lambda x: x[1])
        if c.A == 1:   # one action: log-softmax 0 and probability 1, so the actor's loss is constant: its gradient is exactly 0.0, so is the entropy
            assert not bool(m.grad[: m.n_actor].any()), f"{w}: an actor gradient element is not 0.0 at one action"
            assert float(m._metrics[2]) == 0.0, f"{w}: entropy {float(m._metrics[2])} at one action"
    for m2 in twins:   # with the first handle's form
        ar._opt(b"tensor_core_forward", 1)
        m2.update_from_store(ts, P, 0)
        _states_equal(models[0], m2, f"{what}: a second handle")
    for m in models + twins:
        m.close()
    return worst


def _report(name, c, P, T, blk, ratio):
    print(f"{n_sm()} SMs: {name}: class {c.cls} ({c.kind}, N={c.N}, sharing={c.sharing}/{c.csharing}, D={c.D}, joint={c.joint}, A={c.A}, "
          f"H={c.H}/{c.critic_H}, P={P}, T={T}, {c.N * P * (T + 1)} rows): worst block {blk} at {ratio:.3f} of the {ar.BLOCK_TOL:g} bar")


def _multi(c):
    return c.cls.startswith(("t2", "t3"))


# ---- 1. one case per class ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_the_class_sweep_covers_every_class_on_this_device():
    sm = n_sm()
    actor, critic = set(), set()
    for cls, c in CLASS_CASES.items():
        P, T = shape(dataclasses.replace(c, cls=cls), sm)
        actor |= rp.plan_classes(tuple(rp.nets_of(c.N, c.sharing)), P, T, sm)
        critic |= rp.plan_classes(tuple(rp.nets_of(c.N, c.csharing)), P, T, sm)
    print(f"{sm} SMs: the actor passes cover {len(actor)}, the critic passes {len(critic)} of {len(rp.ALL_CLASSES)} classes")
    assert actor >= set(rp.ALL_CLASSES) and critic >= set(rp.ALL_CLASSES), (sorted(set(rp.ALL_CLASSES) - actor), sorted(set(rp.ALL_CLASSES) - critic))


@pytest.mark.gpu
@pytest.mark.parametrize("cls", list(CLASS_CASES))
@redraw_on_near_tie
def test_class_matches_the_float64_oracle(cls):
    c = dataclasses.replace(CLASS_CASES[cls], cls=cls)
    P, T = shape(c, n_sm())
    blk, ratio = train(c, P, T, f"{cls} ({c.kind}, N={c.N}, P={P}, T={T})", int(torch.randint(0, 1 << 30, (1,))), twin=_multi(c))
    _report(cls, c, P, T, blk, ratio)


# ---- 2. widths and action counts -----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(WIDTH_CASES))
@redraw_on_near_tie
def test_width_matches_the_float64_oracle(name):
    c = WIDTH_CASES[name]
    P, T = shape(c, n_sm())
    blk, ratio = train(c, P, T, f"{name} ({c.cls}, P={P}, T={T})", int(torch.randint(0, 1 << 30, (1,))), twin=True)
    _report(name, c, P, T, blk, ratio)


# ---- 3. episode length -------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(LENGTH_CASES))
@redraw_on_near_tie
def test_episode_length_matches_the_float64_oracle(name):
    c = LENGTH_CASES[name]
    P, T = shape(c, n_sm())
    blk, ratio = train(c, P, T, f"{name} ({c.cls}, P={P}, T={T})", int(torch.randint(0, 1 << 30, (1,))), twin=True)
    _report(name, c, P, T, blk, ratio)


# ---- 4. a handle reused below the shape it was created for ---------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(REUSE_CASES))
@redraw_on_near_tie
def test_handle_reused_at_a_smaller_batch_matches_a_fresh_one(name):
    """a handle created at (2 P, 2 T) trains first on a (2 P, 2 T) store of 1e3-scaled observations, then, parameters reset, on the first P
    environments of a (P, T) store of capacity 2 P at a multi-tile class: the oracle's checks hold and a fresh handle created at (P, T) repeats
    it bit for bit"""
    c = REUSE_CASES[name]
    P, T = shape(c, n_sm())
    seed = int(torch.randint(0, 1 << 30, (1,)))
    warm, _ = data(c, 2 * P, 2 * T, n_sm(), seed + 1)
    warm["obs"] = (warm["obs"] * 1e3).astype(np.float32)
    blk, ratio = train(c, P, T, f"reused {name} handle ({c.cls}, P={P}, T={T})", seed, twin=True, make=(2 * P, 2 * T), warm=warm, cap=2 * P)
    _report(f"reused {name}", c, P, T, blk, ratio)


# ---- 5. the forward kernels at every class of the dense split -------------------------------------------------------------------------------------
FWD_N = ((1, False), (2, False), (3, GROUPS3))
FWD_MAX_ROWS = 51_000              # environments x agents: every class is reached on 114 and 132 SMs
FWD_D, FWD_A = 13, 6
# FP32-only shapes (an input above 32, a hidden width below 128) and the centralised critic read from dense joint rows (row-source mode 3)
FWD_EXTRA = {
    "d100": (Case("ia2c", 2, 100), "t2-c3-part"),
    "h37": (Case("ia2c", 1, FWD_D, H=37, critic_H=37), "t3+-c1-part"),
    "joint16": (Case("maa2c", 2, 8), "t1-c3-part"),
    "joint33": (Case("maa2c", 3, 11, sharing=GROUPS3), "t2-c2-full"),
    "joint128": (Case("mappo", 2, 64), "t3+-c4-part"),
}


def fwd_envs(N, sharing, sm, cls):
    E = rp.find_envs(N, sharing, sm, cls, FWD_MAX_ROWS // N)
    assert E is not None, f"{cls}: no E within {FWD_MAX_ROWS // N} environments reaches it for N={N}, sharing={sharing} on {sm} SMs"
    return E


def _forward_parts(c, m, dqn):
    """(name, call, flat parameters, networks, input width, output width, centralised) of every forward of the handle"""
    if dqn:
        return [("q_values", lambda o: m.q_values(o), m.theta, m.agent_net, c.D, c.A, False),
                ("target q_values", lambda o: m.q_values(o, target=True), m.theta_tgt, m.agent_net, c.D, c.A, False)]
    central = c.kind in CENTRAL and c.N > 1
    return [("logits", lambda o: m.logits(o), m.theta[: m.n_actor], m.actor_net, c.D, c.A, False),
            ("values", lambda o: m.values(o), m.theta[m.n_actor:], m.critic_net, c.joint, 1, central),
            ("target values", lambda o: m.values(o, target=True), m.theta_tgt, m.critic_net, c.joint, 1, central)]


def check_forwards(c, E, what, forms=(1, 0), dqn=False):
    """every forward of an actor-critic (or, dqn, a DQN-family) handle over E environments: each form of tensor_core_forward against the float64
    oracle to 1e-5 of the largest output, the forms against each other on the same bar, a repeated call bit for bit"""
    torch.manual_seed(E + 7 * c.N + c.D)
    if dqn:
        m = ar._dqn_model(ar.Case("idqn", c.N, c.D, A=c.A, sharing=c.sharing, H=c.H, B=4, T=2))
        ar._dqn_perturb(m)
    else:
        m = ar._ac_model(acase(c, 4, 2))
        rac._perturb_target(m)
    obs = torch.randint(-1, 12, (E, c.N, c.D)).float()
    dev = obs.cuda()
    xs = [obs[:, a].double() for a in range(c.N)]
    for name, fwd, flat, nets, ind, outd, central in _forward_parts(c, m, dqn):
        inputs = [obs.reshape(E, c.N * c.D).double()] * c.N if central else xs
        want = torch.stack(gar.agents_forward(flat.detach().cpu().double(), list(nets), inputs, ind, outd), 1).numpy().reshape(E, c.N, outd)
        scale = max(1.0, float(np.abs(want).max()))
        got = {}
        for form in forms:
            ar._opt(b"tensor_core_forward", form)
            a = fwd(dev).clone()
            assert torch.equal(a, fwd(dev)), f"{what}: {name}, tensor_core_forward={form}: a repeated call differs"
            got[form] = a.cpu().numpy().astype(np.float64).reshape(E, c.N, outd)
            err = float(np.abs(got[form] - want).max())
            assert err <= 1e-5 * scale, f"{what}: {name}, tensor_core_forward={form}: max error {err:.3e}, scale {scale:.3g}"
        if len(got) == 2:
            err = float(np.abs(got[1] - got[0]).max())
            assert err <= 1e-5 * scale, f"{what}: {name}, tensor-core vs FP32 forward: max difference {err:.3e}, scale {scale:.3g}"
    m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("cls", list(rp.CLASSES))
def test_forward_class_matches_the_float64_oracle(cls):
    """logits, values and target values of an IA2C handle and the online and target Q-values of an IDQN handle, at the E that reaches the class
    for one agent, two independent agents and three agents in groups (0, 1, 0)"""
    sm = n_sm()
    for N, sharing in FWD_N:
        E = fwd_envs(N, sharing, sm, cls)
        c = Case("ia2c", N, FWD_D, A=FWD_A, sharing=sharing)
        what = f"{cls} forward (N={N}, sharing={sharing}, E={E})"
        check_forwards(c, E, what)
        check_forwards(c, E, what + " DQN", dqn=True)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(FWD_EXTRA))
def test_forward_fp32_shapes_and_joint_rows_match_the_float64_oracle(name):
    """an input of 100 and a hidden width of 37 (the FP32 forward only), and a centralised critic reading dense joint rows at widths 16 (tensor
    cores and FP32), 33 and 128"""
    c, cls = FWD_EXTRA[name]
    E = fwd_envs(c.N, c.sharing, n_sm(), cls)
    forms = (1, 0) if c.H == c.critic_H == 128 and c.joint <= MAX_OBS_TC else (0,)
    check_forwards(c, E, f"{name} forward ({cls}, E={E})", forms)
    if c.kind == "ia2c" and c.D <= MAX_OBS_TC:   # (the DQN family takes inputs up to 32)
        check_forwards(c, E, f"{name} forward ({cls}, E={E}) DQN", (0,), dqn=True)

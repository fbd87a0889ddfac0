"""GPU: the DQN-family training pass (csrc/tc_train.cu's three tensor-core kernels and learner_kernels.cu's fused FP32 train_kernel) at every branch
class of its row split, at 1-8 actions and 1-31 features, and on a handle reused below the shape it was created for, against the float64 oracle.

Which branches of the training pass run depends on how many rows each CTA gets (tests/row_plan.py explains the 24 classes and the two small-net
cases).  The split follows the device's SM count, so the class sweep reads it from the device and picks each case's batch with row_plan.find_batch:
a GPU with another SM count still runs every class.  The episode that ends each CTA has its full length, so the CTA's tail rows -- its last chunk
and the rows of warpgroup 1's after-loop phase -- carry TD errors; the other episodes are ragged.  Each case trains seeded episodes through
update_grads on three handles of the same perturbed parameters (online != target): tensor_core_backward 1, 0, and 1 again.  Checks: the loss and
the filled count; each kernel's gradient against the oracle per parameter block at 1e-5 of the block's largest float64 element; the two kernels
against each other per block; the second tensor-core handle repeats the first bit for bit.  QMIX cases run marl_dqn_update and
tests/test_qmix_agents_gpu.py's per-update checks.

The TD head reaches the training pass from four sources, spread over the classes: the in-kernel head (IDQN; double-Q only where a CTA holds few
rows, as tests/test_agent_range.py requires), td_ext with stride 0 (VDN), per-agent td_ext (IDQN with standardise_returns) and the QMIX mixer.

tests/test_row_plan.py checks without a GPU that every case still finds its class on 114 and 132 SMs and sits on the edge it claims."""
import copy
import dataclasses

import numpy as np
import pytest
import torch

from oracle import learner_ref as lr
from oracle import qmix_ref as qr
from tests import qmix_options_ref as qo
from tests import row_plan as rp
from tests import test_agent_range_gpu as ar
from tests import test_qmix_agents_gpu as qa
from tests.helpers import assert_grad_close, redraw_on_near_tie, traj_store

MAX_ROWS = 20_000          # rows N B (T + 1) per case: the float64 oracle stays quick
MAX_OBS_TC = 32            # kMaxObsDim: the tensor-core backward takes D < 32 (column D carries the bias)
TS_ALL = tuple(range(8, 400))    # up to 3+ tiles of one episode per CTA; T >= 8 keeps a few TD errors per episode (one is ill-conditioned)
TS_SHORT = tuple(range(4, 64))   # several episodes per CTA (min_units >= 2)
TS_MANY = tuple(range(20, 64))   # a few hundred episodes: several per CTA at a multi-tile class, tile boundaries inside an episode
SEPS = ar.SEPS             # 16 agents in groups of 13 / 2 / 1, interleaved
GROUPS4 = (0, 1, 0, 0)     # 4 agents in groups of 3 / 1


@dataclasses.dataclass(frozen=True)
class Case:
    kind: str                    # idqn, vdn, qmix
    N: int
    D: int
    A: int = 6
    sharing: object = False      # False, True or a tuple of group labels (QMIX: False or True)
    double_q: bool = False
    standardise: bool = False
    T_choices: tuple = TS_ALL
    cls: str = None              # the width sweep: the class its case runs at


CLASS_CASES = {
    "t1-c1-full": Case("idqn", 1, 12, double_q=True, T_choices=TS_SHORT),
    "t1-c1-part": Case("vdn", 3, 6, sharing=True),
    "t1-c2-full": Case("idqn", 2, 15, standardise=True),
    "t1-c2-part": Case("qmix", 3, 9),
    "t1-c3-full": Case("idqn", 4, 30, sharing=GROUPS4),
    "t1-c3-part": Case("idqn", 2, 5, double_q=True),
    "t1-c4-full": Case("vdn", 2, 11),
    "t1-c4-part": Case("idqn", 16, 10, sharing=SEPS),
    "t2-c1-full": Case("idqn", 1, 20, double_q=True),
    "t2-c1-part": Case("idqn", 4, 7, sharing=True, double_q=True),
    "t2-c2-full": Case("idqn", 3, 13, standardise=True),
    "t2-c2-part": Case("idqn", 4, 30, sharing=True, T_choices=TS_MANY),
    "t2-c3-full": Case("qmix", 2, 14, sharing=True),
    "t2-c3-part": Case("idqn", 1, 4, T_choices=TS_MANY),
    "t2-c4-full": Case("vdn", 5, 18),
    "t2-c4-part": Case("idqn", 2, 23),
    "t3+-c1-full": Case("idqn", 1, 30),
    "t3+-c1-part": Case("vdn", 2, 12, sharing=True),
    "t3+-c2-full": Case("idqn", 4, 6, sharing=GROUPS4),
    "t3+-c2-part": Case("idqn", 2, 19, standardise=True),
    "t3+-c3-full": Case("qmix", 4, 10),
    "t3+-c3-part": Case("idqn", 3, 27),
    "t3+-c4-full": Case("vdn", 6, 15),
    "t3+-c4-part": Case("idqn", 1, 29),
    rp.SMALL_NET: Case("idqn", 2, 3, double_q=True),
    rp.ONE_CTA: Case("vdn", 2, 8, sharing=True),
}

# the k1steps edges of layer1_tile (D = 8 k - 1, 8 k, 8 k + 1; at 8, 16 and 24 the ones line of [X | 1] opens a new 8-line group), each with an
# action count: 1 (no argmax; db3[0] only), 2 and 5 (partial head_quad / wgmma_ss_n8 columns), 3, 8 (kOutPad)
WIDTH_CASES = {
    "d1_a1": Case("idqn", 2, 1, A=1, double_q=True, cls="t2-c1-part"),
    "d2_a2": Case("vdn", 2, 2, A=2, cls="t2-c2-part"),
    "d7_a3": Case("idqn", 2, 7, A=3, cls="t2-c3-part"),
    "d8_a5": Case("idqn", 3, 8, A=5, sharing=True, cls="t2-c4-part"),
    "d9_a8": Case("idqn", 2, 9, A=8, cls="t3+-c1-part"),
    "d16_a1": Case("vdn", 2, 16, A=1, double_q=True, cls="t3+-c2-part"),
    "d17_a2": Case("idqn", 2, 17, A=2, standardise=True, cls="t3+-c3-part"),
    "d24_a3": Case("idqn", 4, 24, A=3, sharing=GROUPS4, cls="t3+-c4-part"),
    "d25_a5": Case("vdn", 3, 25, A=5, cls="t2-c1-part"),
    "d31_a8": Case("idqn", 2, 31, A=8, cls="t2-c3-part"),
}

FWD_E = (1, 9001)   # one env, and a ragged split of more than 128 rows per CTA on 114 and 132 SMs

# handle reuse: (max_batch, max_T) it is created at, (B, T) it then trains on
REUSE_SHAPES = {"idqn": ((24, 40), (9, 17)), "vdn": ((20, 33), (7, 12)), "qmix": ((16, 30), (5, 11))}
REUSE_CASES = {"idqn": Case("idqn", 3, 10), "vdn": Case("vdn", 4, 7, sharing=True), "qmix": Case("qmix", 3, 9)}


def _n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(autouse=True)
def _restore():
    yield
    ar._opt(b"tensor_core_backward", True)   # the library defaults
    ar._opt(b"tensor_core_forward", True)


def _shape(c, cls):
    """(B, T) of the case on this device; a class out of reach fails (a device with another SM count must not quietly test less)"""
    n_sm = _n_sm()
    found = rp.find_batch(c.N, c.sharing, c.T_choices, n_sm, cls, MAX_ROWS)
    assert found is not None, f"{cls}: no batch of {c} within {MAX_ROWS} rows reaches it on {n_sm} SMs"
    print(f"{n_sm} SMs: class {cls}: N={c.N} sharing={c.sharing} B={found[0]} T={found[1]}")
    return found


def _acase(c, B, T):
    return ar.Case(c.kind, c.N, c.D, A=c.A, sharing=c.sharing, B=B, T=T, double_q=c.double_q, standardise=c.standardise)


def _check_stats(m, g, fill, want, what):
    n = m.n_params
    assert g[n + 1] == fill, f"filled count, {what}: {g[n + 1]} vs {fill}"
    loss = float(g[n]) / fill
    assert abs(loss - want["loss"]) <= 1e-5 * max(1.0, abs(want["loss"])), f"loss, {what}: {loss} vs {want['loss']}"


def _td_floors(ac, m, st, b, hp):
    """Every gradient block of net k is a sum over its rows of g_r x dq_r[act_r]/dtheta, g_r = dL/dq_r[act_r] = 2 delta_r filled_r / filled.  Where
    the TD errors of the rows cancel -- at one action and a one-feature input every row's dq/dtheta is nearly the same -- that sum is far smaller
    than the terms a float32 reduction rounds.  A block's scale is then the same sum with |g_r|, in float64 (as test_agent_range_gpu's
    _critic_bias_floors for the critic's bias).  None with standardise_returns, whose statistics would have to be stepped first."""
    if ac.standardise:
        return None
    obs, act, rew, done, filled = (b[k] for k in ("obss", "actions", "rewards", "dones", "filled"))
    th = st.theta.clone().requires_grad_(True)
    q = torch.stack(lr.agents_forward(th, st.agent_net, list(obs), ac.D, ac.A))                        # (N, T + 1, B, A)
    with torch.no_grad():
        tq = torch.stack(lr.agents_forward(st.theta_tgt, st.agent_net, list(obs), ac.D, ac.A))[:, 1:]
        nxt = tq.gather(-1, q[:, 1:].argmax(-1, keepdim=True)).squeeze(-1) if hp.double_q else tq.max(-1)[0]
    chosen = q[:, :-1].gather(-1, act.unsqueeze(-1)).squeeze(-1)                                     # (N, T, B)
    with torch.no_grad():
        if ac.kind == "vdn":
            delta = (chosen.sum(0) - (rew[0] + hp.gamma * nxt.sum(0) * (1 - done[1:]))).expand_as(chosen)
        else:
            delta = chosen - (rew + hp.gamma * nxt * (1 - done[1:]))
        g = (2 * delta * filled / filled.sum()).abs()
    (grad,) = torch.autograd.grad((g * chosen).sum(), th)
    return {name: float(grad[sl].abs().max()) for name, sl in ar._blocks(m)}


def _tail_episodes(c, B, T):
    """the episodes that end a CTA on this device: given their full length T, the tail rows of every CTA carry TD errors (row_plan.py)"""
    return rp.last_episodes(rp.nets_of(c.N, c.sharing), B, T, _n_sm())


def _train_dqn(c, B, T, what):
    """IDQN / VDN: update_grads on a tensor-core handle, an FP32 handle and a second tensor-core handle of the same parameters"""
    ac = _acase(c, B, T)
    hp = ar._dqn_hp(ac)
    models = [ar._dqn_model(ac) for _ in range(3)]
    ar._dqn_perturb(models[0])
    for m in models[1:]:
        ar._dqn_copy(m, models[0])
    st = ar._dqn_oracle(ac, models[0])
    s = ar._dqn_store(ac, int(torch.randint(0, 1 << 30, (1,))))
    full = _tail_episodes(c, B, T)
    s["filled"][full] = 1; s["done"][full] = 0; s["done"][full, T] = 1
    b64 = ar._f64(lr.batch_from_store(s, np.arange(B)))
    ar._dqn_margin(ac, st, b64, hp)
    st0 = copy.deepcopy(st)
    want = lr.dqn_update(st, b64, hp)
    ts = traj_store(s, models[0].device)
    idx = torch.arange(B, dtype=torch.int32, device=models[0].device)
    fill = float(b64["filled"].sum())
    kink = lambda: lr.dqn_kink_risk(st0, b64, hp)   # noqa: E731
    floors = _td_floors(ac, models[0], st0, b64, hp)
    grads = []
    for form, m in zip((1, 0, 1), models):
        ar._opt(b"tensor_core_backward", form)
        m.update_grads(ts, idx)
        g = m.grad.cpu().numpy()
        grads.append(g)
        w = f"{what}, tensor_core_backward={form}"
        _check_stats(m, g.astype(np.float64), fill, want, w)
        blk, ratio = ar._assert_blocks(m, g[: m.n_params].astype(np.float64) / fill, want["grad"].numpy(), w, kink, floors=floors)
        print(f"{w}: worst gradient block {blk} at {ratio:.3f} of the {ar.BLOCK_TOL:g} bar")
    n = models[0].n_params
    blk, ratio = ar._assert_blocks(models[0], grads[0][:n].astype(np.float64) / fill, want["grad"].numpy(), f"{what}: tensor-core vs FP32", kink,
                                   other=grads[1][:n].astype(np.float64) / fill, floors=floors)
    print(f"{what}: tensor-core vs FP32, worst block {blk} at {ratio:.3f} of the bar")
    assert np.array_equal(grads[0], grads[2]), f"{what}: a second tensor-core handle differs from the first"
    for m in models:
        m.close()


def _qcase(c, B, T):
    return qa.Case(N=c.N, D=c.D, T=T, B=B, sharing=c.sharing, double_q=c.double_q)


def _train_qmix(c, B, T, what, monkeypatch):
    """QMIX: marl_dqn_update on the same three handles, each through test_qmix_agents_gpu's per-update checks"""
    qc = _qcase(c, B, T)
    hp = qa._hp(qc)
    models = [qa._model(qc, monkeypatch) for _ in range(3)]
    qa._perturb_target(models[0])
    for m in models[1:]:
        qa._copy_params(models[0], m)
    st = qa._oracle(qc, models[0])
    batch = qr.random_batch(c.N, T, B, c.D, qa.A, seed=int(torch.randint(0, 1 << 30, (1,))), ragged=True)
    full = _tail_episodes(c, B, T)
    batch["filled"][:, full] = 1.0; batch["dones"][:, full] = 0.0; batch["dones"][T, full] = 1.0
    b64 = qa._f64(batch)
    qa._margin(qc, st, b64, hp)
    st0 = copy.deepcopy(st)
    want = qo.qmix_update(st, b64, hp)
    ts = qa._to_store(batch, models[0].device)
    idx = torch.arange(B, dtype=torch.int32, device=models[0].device)
    fill = float(b64["filled"].sum())
    for form, m in zip((1, 0, 1), models):
        ar._opt(b"tensor_core_backward", form)
        met = m.update_from_store(ts, idx).cpu()
        blk, ratio = qa._check_update(qc, m, st, st0, b64, want, met, hp, f"{what}, tensor_core_backward={form}", per_block=True)
        print(f"{what}, tensor_core_backward={form}: worst mixer block {blk} at {ratio:.3f} of the bar")
    n = models[0].n_params
    g0, g1 = (m.grad.cpu().numpy()[:n].astype(np.float64) / fill for m in models[:2])
    blk, ratio = ar._assert_blocks(models[0], g0, want["grad"].numpy(), f"{what}: tensor-core vs FP32", lambda: qo.qmix_kink_risk(st0, b64, hp), other=g1)
    print(f"{what}: tensor-core vs FP32, worst agents' block {blk} at {ratio:.3f} of the bar")
    a, b = qa._state(models[0]), qa._state(models[2])
    for k in a:
        assert torch.equal(a[k], b[k]), f"{what}: {k} differs between two tensor-core handles"
    for m in models:
        m.close()


# ---- 1. one case per class ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_the_class_sweep_covers_every_class_on_this_device():
    n_sm = _n_sm()
    covered = set()
    for cls, c in CLASS_CASES.items():
        B, T = _shape(c, cls)
        covered |= rp.plan_classes(tuple(rp.nets_of(c.N, c.sharing)), B, T, n_sm)
    print(f"{n_sm} SMs: the class sweep covers {len(covered & set(rp.ALL_CLASSES))} of {len(rp.ALL_CLASSES)} classes: {sorted(covered)}")
    assert covered >= set(rp.ALL_CLASSES), sorted(set(rp.ALL_CLASSES) - covered)


@pytest.mark.gpu
@pytest.mark.parametrize("cls", list(CLASS_CASES))
@redraw_on_near_tie
def test_class_matches_the_float64_oracle(cls, monkeypatch):
    c = CLASS_CASES[cls]
    B, T = _shape(c, cls)
    what = f"{cls} ({c.kind}, N={c.N}, D={c.D}, B={B}, T={T})"
    if c.kind == "qmix":
        _train_qmix(c, B, T, what, monkeypatch)
    else:
        _train_dqn(c, B, T, what)


# ---- 2. widths and action counts -----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(WIDTH_CASES))
@redraw_on_near_tie
def test_width_matches_the_float64_oracle(name):
    c = WIDTH_CASES[name]
    B, T = _shape(c, c.cls)
    _train_dqn(c, B, T, f"{name} ({c.cls}, {c.kind}, N={c.N}, B={B}, T={T})")


@pytest.mark.gpu
@pytest.mark.parametrize("E", FWD_E)
@pytest.mark.parametrize("name", list(WIDTH_CASES))
def test_width_q_values_match_the_oracle(name, E):
    """q_values of online and target networks: the tensor-core and the FFMA forward against the float64 oracle and each other, to 1e-5 of the
    largest |Q|"""
    c = WIDTH_CASES[name]
    torch.manual_seed(c.D * 10 + c.A)
    m = ar._dqn_model(_acase(c, 4, 2))
    ar._dqn_perturb(m)
    obs = torch.randint(-1, 12, (E, c.N, c.D)).float()
    xs = [obs[:, a].double() for a in range(c.N)]
    for target, flat in ((False, m.theta), (True, m.theta_tgt)):
        want = torch.stack(lr.agents_forward(flat.cpu().double(), list(m.agent_net), xs, c.D, c.A), 1).numpy()
        got = {}
        for tc in (1, 0):
            ar._opt(b"tensor_core_forward", tc)
            got[tc] = m.q_values(obs.cuda(), target=target).cpu().numpy().astype(np.float64)
        scale = max(1.0, float(np.abs(want).max()))
        for what, a, b in (("tensor-core", got[1], want), ("FFMA", got[0], want), ("tensor-core vs FFMA", got[1], got[0])):
            err = float(np.abs(a - b).max())
            assert err <= 1e-5 * scale, f"{name}, E={E}: {what} q_values (target={target}): max error {err:.3e}, scale {scale:.3g}"
    m.close()


# ---- 3. a handle reused below the shape it was created for ---------------------------------------------------------------------------------------
def _reuse_model(kind, c, B, T, monkeypatch):
    if kind == "qmix":
        return qa._model(_qcase(c, B, T), monkeypatch)
    return ar._dqn_model(_acase(c, B, T))


def _reuse_batch(kind, c, B, T, seed, scale=1.0):
    """(oracle batch, device store) of B seeded ragged episodes of T steps; observations and rewards times `scale`"""
    if kind == "qmix":
        b = qr.random_batch(c.N, T, B, c.D, qa.A, seed=seed, ragged=True)
        b["obss"] = b["obss"] * scale; b["rewards"] = b["rewards"] * scale
        return b, qa._to_store(b, "cuda")
    s = ar._dqn_store(_acase(c, B, T), seed)
    s["obs"] = (s["obs"] * scale).astype(np.float32); s["rew"] = (s["rew"] * scale).astype(np.float32)
    return lr.batch_from_store(s, np.arange(B)), traj_store(s, "cuda")


def _params(kind, m):
    names = ("theta", "theta_tgt") + (("mix", "mix_tgt") if kind == "qmix" else ())
    return {k: getattr(m, k).detach().clone() for k in names}


def _set_params(m, p):
    for k, v in p.items():
        getattr(m, k).copy_(v)
    m.params_changed()


def _grads(kind, m):
    return [m.grad.cpu()] + ([m.mix_grad.cpu()] if kind == "qmix" else [])


@pytest.mark.gpu
@pytest.mark.parametrize("tc", [1, 0])
@pytest.mark.parametrize("kind", list(REUSE_CASES))
@redraw_on_near_tie
def test_handle_reused_at_a_smaller_batch_matches_a_fresh_one(kind, tc, monkeypatch):
    """A handle created at (max_batch, max_T) trains on a (max_batch, max_T) batch whose observations and rewards are scaled by 1e3 (every
    intermediate buffer then holds large values), then, parameters reset, on a smaller (B, T) batch: its gradient and loss statistics are those of
    a fresh handle created at (B, T), bit for bit, and meet the oracle"""
    c = REUSE_CASES[kind]
    (Bm, Tm), (B, T) = REUSE_SHAPES[kind]
    ar._opt(b"tensor_core_backward", tc)
    big = _reuse_model(kind, c, Bm, Tm, monkeypatch)
    (qa._perturb_target if kind == "qmix" else ar._dqn_perturb)(big)
    fresh = _reuse_model(kind, c, B, T, monkeypatch)
    p0 = _params(kind, big)
    _set_params(fresh, p0)
    seed = int(torch.randint(0, 1 << 30, (1,)))
    _, ts_big = _reuse_batch(kind, c, Bm, Tm, seed + 1, scale=1e3)
    big.update_grads(ts_big, torch.arange(Bm, dtype=torch.int32, device="cuda"))
    assert all(bool(torch.isfinite(g).all()) for g in _grads(kind, big))
    _set_params(big, p0)
    batch, ts = _reuse_batch(kind, c, B, T, seed)
    idx = torch.arange(B, dtype=torch.int32, device="cuda")
    big.update_grads(ts, idx)
    fresh.update_grads(ts, idx)
    for name, a, b in zip(("grad", "mixer grad"), _grads(kind, big), _grads(kind, fresh)):
        assert torch.equal(a, b), f"{kind}, tensor_core_backward={tc}: {name} of the reused handle differs from a fresh one " \
                                  f"(max abs difference {float((a.double() - b.double()).abs().max()):.3e})"
    b64 = ar._f64(batch)
    fill = float(b64["filled"].sum())
    what = f"reused {kind} handle, tensor_core_backward={tc}"
    g = fresh.grad.cpu().numpy().astype(np.float64)
    if kind == "qmix":
        qc = _qcase(c, B, T)
        hp = qa._hp(qc)
        st = qa._oracle(qc, fresh)
        qa._margin(qc, st, b64, hp)
        st0 = copy.deepcopy(st)
        want = qo.qmix_update(st, b64, hp)
        _check_stats(fresh, g, fill, want, what)
        assert_grad_close(lr, st0, b64, hp, g[: fresh.n_params] / fill, want["grad"].numpy(), tol=2e-5, what=f"agents' gradient, {what}",
                          kink_risk=lambda: qo.qmix_kink_risk(st0, b64, hp))   # the bar of test_qmix_agents_gpu's _check_update
        qa._assert_blocks(qc, fresh.mix_grad[: fresh.n_mix].cpu().numpy() / fill, want["mix_grad"].numpy(), what)
    else:
        ac = _acase(c, B, T)
        hp = ar._dqn_hp(ac)
        st = ar._dqn_oracle(ac, fresh)
        ar._dqn_margin(ac, st, b64, hp)
        st0 = copy.deepcopy(st)
        want = lr.dqn_update(st, b64, hp)
        _check_stats(fresh, g, fill, want, what)
        blk, ratio = ar._assert_blocks(fresh, g[: fresh.n_params] / fill, want["grad"].numpy(), what, lambda: lr.dqn_kink_risk(st0, b64, hp),
                                       floors=_td_floors(ac, fresh, st0, b64, hp))
        print(f"{what}: worst gradient block {blk} at {ratio:.3f} of the {ar.BLOCK_TOL:g} bar")
    big.close(); fresh.close()

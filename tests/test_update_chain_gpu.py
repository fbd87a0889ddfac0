"""GPU: the multi-update DQN learner path -- marl_dqn_update_n (on-device replay sampling, the fused reduce + Adam tail, weight images kept
current by the Adam step, state carried from one update to the next) -- which every IDQN / VDN / QMIX training run spends its time in.

1. update_n is bit-for-bit the loop it replaces: replay_sample + update_from_store, K times.
2. K fused single updates (update_from_store) against the oracle, never glued: the device state evolves on its own, the oracle in step with it.
3. The packed images the Adam step keeps current are the images a full repack (params_changed) produces.

Block shapes of reduce_adam_kernel<0> on 132 SMs (one block per SM), obs width 15 unless stated: 1 network -> 160 parameters per block x 4 slices,
2 -> 320 x 3, 3 (obs 27) -> 480 x 2, 4 -> more than 512: the two-kernel tail (grad_reduce_kernel + adam_kernel)."""
import copy
import ctypes as C
import dataclasses
import types

import numpy as np
import pytest
import torch

from oracle import learner_ref as lr
from oracle import policy_ref
from oracle import qmix_ref as qr
from tests.helpers import assert_grad_close, check_margin, close_scaled, random_store, redraw_on_near_tie, space

pytestmark = pytest.mark.gpu
A = 6
MIXING = dict(embed_dim=64, hypernet_layers=2, hypernet_embed=32)
SEED = 0x5EED_1234_ABCD


@dataclasses.dataclass(frozen=True)
class Case:
    mixer: int = 0               # 0 IDQN, 1 VDN, 2 QMIX
    N: int = 2
    D: int = 15
    sharing: object = False
    B: int = 64                  # batch = max_batch
    T: int = 25
    tu: float = 3                # target_update_interval_or_tau
    grad_clip: float = 1.0       # None: no clipping
    double_q: bool = False
    K: int = 8                   # updates in the chain
    first: int = 0               # update index of the first update (Philox counter)
    cap: int = 300
    n_valid: int = 300
    standardise: bool = False
    tc_backward: bool = True


# Each case covers something no other case does.  Test 2 compares K-step chains with the oracle; a double-Q argmax near-tie anywhere in the chain
# re-draws the case, so double-Q runs only where the chain has few rows (batch 1) or few steps (K = 4); hard syncs every 3 updates: K = 8 crosses two.
CASES = {
    # fused tail 320 x 3; the chain's update index crosses the high word of the Philox counter
    "idqn2_b256_philox_high_word": Case(B=256, first=2**32 - 3),
    # fused tail 160 x 4, Polyak target, no clipping, a batch of one episode
    "idqn_shared_polyak_noclip_b1": Case(sharing=True, B=1, tu=0.05, grad_clip=None, double_q=True),
    # fused tail 480 x 2; batch 33 (not a multiple of 4: the k & 3 pick of the Philox word); n_valid below capacity and not a power of two
    "idqn3_obs27_b33_nvalid257": Case(N=3, D=27, B=33, n_valid=257),
    # 4 networks: the two-kernel tail inside marl_dqn_update
    "idqn4_two_kernel_tail": Case(N=4, B=48, T=12),
    # running return statistics carried across fused updates (VDN keeps one per batch entry: batch = max_batch)
    "vdn2_standardise_returns": Case(mixer=1, B=48, standardise=True),
    # the same above 64 batch entries: one statistics column per entry of 25 returns, whose moments ret_moments_cols_kernel takes
    "vdn2_standardise_returns_b128": Case(mixer=1, B=128, standardise=True),
    # the mixer's gradient and Adam step next to the fused tail; hard syncs of the target mixer (single-Q: a double-Q chain of this length tied in
    # 3 of 5 initialisations; tests/test_qmix.py compares the mixer's double-Q target with the oracle)
    "qmix2": Case(mixer=2, B=32, K=8, T=10),
    # widest observation of the tensor-core backward; the double-Q chain (K = 4, 32 x 10 steps)
    "idqn2_obs31_double_q": Case(D=31, B=32, T=10, double_q=True, K=4),
    # observation width 32: the FP32 train kernel inside the chain
    "idqn2_obs32": Case(D=32, B=64),
    # the FP32 training pass (tensor_core_backward = 0) with the fused tail; clipping active on every update
    "idqn2_ffma_train_clip_active": Case(B=64, grad_clip=0.05, tc_backward=False),
}


def _opt(name, on):
    from codebase_b200 import _native as nat

    nat.check(nat.lib().marl_set_option(name, C.c_int32(int(on))), "marl_set_option")


@pytest.fixture(autouse=True)
def _restore():
    yield
    _opt(b"tensor_core_backward", True)   # the library defaults
    _opt(b"tensor_core_forward", True)


def _hp(c):
    return lr.DqnHP(grad_clip=c.grad_clip, double_q=c.double_q, target_update_interval_or_tau=c.tu, mixer=c.mixer)


def _learner(c):
    from codebase_b200.dqn import model as M

    hp = _hp(c)
    cfg = types.SimpleNamespace(optimizer="Adam", lr=hp.lr, gamma=hp.gamma, grad_clip=c.grad_clip, double_q=c.double_q, target_update_interval_or_tau=c.tu,
                                standardise_returns=c.standardise)
    args = ([space(shape=(c.D,))] * c.N, [space(n=A)] * c.N, cfg, [128, 128], c.sharing, False, True)
    if c.mixer == 2:
        return M.QMixNetwork(*args, MIXING, "cuda", max_batch=c.B, max_episode_length=c.T)
    return (M.VDNetwork if c.mixer else M.QNetwork)(*args, "cuda", max_batch=c.B, max_episode_length=c.T)


def _perturb_target(m):
    """a target that differs from the online networks until the first hard sync, so that the target networks' images matter"""
    m.theta_tgt.copy_(m.theta + 0.01 * torch.randn_like(m.theta))
    if m.mixer == 2:
        m.mix_tgt.copy_(m.mix + 0.01 * torch.randn_like(m.mix))
    m.params_changed()


def _copy_params(dst, src):
    dst.theta.copy_(src.theta); dst.theta_tgt.copy_(src.theta_tgt)
    if src.mixer == 2:
        dst.mix.copy_(src.mix); dst.mix_tgt.copy_(src.mix_tgt)
    dst.params_changed()


def _device_store(s, c, device):
    from codebase_b200.lbf import TrajStore

    ts = TrajStore(c.cap, c.N, c.T, c.D, device)
    for k in ("obs", "act", "rew", "done", "filled"):
        getattr(ts, k).copy_(torch.as_tensor(s[k]))
    return ts


def _counters(m):
    """(updates, last_target_update)"""
    from codebase_b200 import _native as nat

    u, last = C.c_int64(), C.c_int64()
    nat.check(m._lib.marl_dqn_counters(m._h, C.byref(u), C.byref(last)), "marl_dqn_counters")
    return int(u.value), int(last.value)


def _state(m):
    """everything an update reads or writes, for bitwise comparison"""
    out = dict(theta=m.theta, theta_tgt=m.theta_tgt, adam_m=m.adam_m, adam_v=m.adam_v, grad=m.grad, metrics=m._metrics)
    if m.mixer == 2:
        out.update(mix=m.mix, mix_tgt=m.mix_tgt, mix_m=m.mix_m, mix_v=m.mix_v, mix_grad=m.mix_grad)
    out = {k: v.detach().cpu().clone() for k, v in out.items()}
    if m.standardise_returns:
        mean, var, count = m.ret_ms()
        out.update(ret_mean=mean, ret_var=var, ret_count=torch.tensor(count, dtype=torch.float64))
    return out


# ---- 1. update_n == K x (replay_sample, update_from_store), bit for bit ------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(CASES))
def test_update_n_is_the_loop_it_replaces(case):
    """Same deterministic kernels on the same inputs: any difference is a defect of the on-device sampling (the next update's indices drawn in the
    tail kernel), the launch chain, or the image / target bookkeeping between updates."""
    from codebase_b200 import _native as nat

    c = CASES[case]
    _opt(b"tensor_core_backward", c.tc_backward)
    torch.manual_seed(3)
    a = _learner(c)
    _perturb_target(a)
    b = _learner(c)
    _copy_params(b, a)
    rng = np.random.default_rng(c.B * 31 + c.D)
    ts = _device_store(random_store(rng, c.cap, c.N, c.T, c.D, c.mixer != 0), c, a.device)

    a.update_n(ts, c.B, c.n_valid, SEED, c.first, c.K)
    idx = torch.zeros(c.B, dtype=torch.int32, device=b.device)
    for u in range(c.K):
        nat.check(nat.lib().marl_replay_sample(C.c_uint64(SEED), C.c_uint64(c.first + u), C.c_int32(c.B), C.c_int32(c.n_valid), nat.ptr(idx), nat.stream_ptr()), "sample")
        assert np.array_equal(idx.cpu().numpy(), policy_ref.replay_sample(SEED, c.first + u, c.B, c.n_valid)), f"replay indices of update {u}"
        b.update_from_store(ts, idx)
    got, want = _state(a), _state(b)
    assert got.keys() == want.keys()
    for k in want:
        assert torch.equal(got[k], want[k]), f"{k}: max abs difference {float((got[k].double() - want[k].double()).abs().max()):.3e}"
    assert a.updates == b.updates == c.K
    assert _counters(a) == _counters(b)
    a.close(); b.close()


# ---- 2. the fused single-update chain against the oracle, never glued ----------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(CASES))
@redraw_on_near_tie
def test_fused_chain_matches_oracle(case):
    """K updates through marl_dqn_update (the fused tail) with the oracle's replay indices; the device's parameters, Adam state, targets, counters
    and running statistics are never overwritten.  The oracle (lr.dqn_update / qr.qmix_update) takes the same batches in step.  With test 1 this
    pins update_n, the path of every training run."""
    c = CASES[case]
    _opt(b"tensor_core_backward", c.tc_backward)
    hp = _hp(c)
    m = _learner(c)
    _perturb_target(m)
    agent_net = list(m.agent_net)
    if c.mixer == 2:
        st = qr.QmixState(m.theta.cpu().clone(), m.theta_tgt.cpu().clone(), m.mix.cpu().clone(), m.mix_tgt.cpu().clone(), agent_net, c.D, A)
    else:
        ret_ms = lr.RunningMeanStdRef((1,) if c.mixer else (c.N,)) if c.standardise else None
        st = lr.DqnState(m.theta.cpu().clone(), m.theta_tgt.cpu().clone(), agent_net, c.D, A, ret_ms=ret_ms)
    rng = np.random.default_rng(c.B * 31 + c.D)
    s = random_store(rng, c.cap, c.N, c.T, c.D, c.mixer != 0)
    ts = _device_store(s, c, m.device)
    n = m.n_params
    # gradient bars (and Adam's m / v, which follow the gradient): QMIX's are those of tests/test_qmix.py::test_gpu_update_matches_oracle (the
    # mixer's FP32 arithmetic), the standardised loss's those of tests/test_standardise_returns_dqn.py::test_device_matches_oracle; every other
    # bar, the loss of every case included, is BASELINE.json's 1e-5
    gtol = 2e-5 if c.mixer == 2 or c.standardise else 1e-5
    for u in range(c.K):
        idx = policy_ref.replay_sample(SEED, c.first + u, c.B, c.n_valid)
        batch = lr.batch_from_store(s, idx)
        if c.double_q:   # a near-tie makes the comparison a coin toss: re-drawn by the decorator
            check_margin(lr, lr.DqnState(st.theta, st.theta_tgt, agent_net, c.D, A) if c.mixer == 2 else st, batch, hp)
        st0 = copy.deepcopy(st)   # the oracle steps st in place; a ReLU kink is judged on the state before the update
        want = qr.qmix_update(st, batch, hp) if c.mixer == 2 else lr.dqn_update(st, batch, hp)
        met = m.update_from_store(ts, torch.tensor(idx, device=m.device)).cpu().numpy()
        g = m.grad.cpu().numpy()
        fill = float(batch["filled"].sum())
        assert g[n + 1] == fill and met[4] == fill, (u, g[n + 1], met[4], fill)
        what = f"update {u}:"
        risk = (lambda: qr.qmix_kink_risk(st0, batch, hp)) if c.mixer == 2 else None
        assert_grad_close(lr, st0, batch, hp, g[:n] / g[n + 1], want["grad"].numpy(), tol=gtol, what=what, kink_risk=risk)
        if c.mixer == 2:   # no kink excuse for the mixer's own gradient, as in tests/test_qmix.py
            assert_grad_close(lr, st0, batch, hp, m.mix_grad[: m.n_mix].cpu().numpy() / fill, want["mix_grad"].numpy(), tol=gtol, what=f"{what} mixer",
                              kink_risk=lambda: 0.0)
        assert abs(met[0] - want["loss"]) <= 1e-5 * max(1.0, abs(want["loss"])), (what, met[0], want["loss"])
        # the global norm of the clip, from the per-block sums of squares inside the tail kernel
        assert np.allclose(met[1], want["grad_norm"], rtol=1e-4, atol=1e-5), (what, met[1], want["grad_norm"])
        if c.grad_clip is not None and c.grad_clip < 0.1:
            assert want["grad_norm"] > c.grad_clip, "this case is meant to clip on every update"
        close_scaled(m.adam_m.cpu().numpy(), st.m.numpy(), gtol); close_scaled(m.adam_v.cpu().numpy(), st.v.numpy(), 2 * gtol)
        pairs = [("theta", m.theta, st.theta), ("theta_tgt", m.theta_tgt, st.theta_tgt)]
        if c.mixer == 2:
            close_scaled(m.mix_m.cpu().numpy(), st.mix_m.numpy(), gtol); close_scaled(m.mix_v.cpu().numpy(), st.mix_v.numpy(), 2 * gtol)
            pairs += [("mix", m.mix, st.mix), ("mix_tgt", m.mix_tgt, st.mix_tgt)]
        for name, mine, theirs in pairs:
            d = np.abs(mine.cpu().numpy() - theirs.numpy())
            assert np.quantile(d, 0.999) < (2e-5 if c.mixer == 2 else 1e-5) and d.max() < 2 * hp.lr * (u + 1) + 1e-6, (what, name, np.quantile(d, 0.999), d.max())
        if c.standardise:
            mean, var, count = m.ret_ms()
            for got, ref in ((mean, st.ret_ms.mean), (var, st.ret_ms.var)):
                ref = ref.numpy() if ref.numel() > 1 else np.full(len(got), float(ref))
                assert np.allclose(got.numpy(), ref, rtol=1e-5, atol=1e-5), (what, float(np.abs(got.numpy() - ref).max()))
            assert abs(count - st.ret_ms.count) < 1e-6, (what, count, st.ret_ms.count)
        assert _counters(m) == (st.updates, st.last_target_update), (what, _counters(m), st.updates, st.last_target_update)
    if c.tu > 1:
        assert st.last_target_update == c.K // int(c.tu) * int(c.tu) > 0
    m.close()


# ---- 3. images kept current by the Adam step == a full repack --------------------------------------------------------------------------------------
# (case, phases): one update_n call per phase, (updates, tensor_core_forward, tensor_core_backward); the check then runs with both options on
IMAGE_CASES = {
    "idqn2_ends_on_hard_sync": (Case(), [(4, 1, 1), (2, 1, 1)]),                   # update 6 is the second hard sync
    "idqn2_one_after_hard_sync": (Case(), [(7, 1, 1)]),
    "idqn_shared_polyak": (Case(sharing=True, tu=0.05), [(5, 1, 1)]),
    "idqn4_tc_forward_off_midway": (Case(N=4, B=48, T=12), [(2, 1, 1), (3, 0, 1), (2, 1, 1)]),   # the two-kernel tail's adam_kernel
    # the chain ends with tensor_core_forward = 0: the Adam steps left the online images alone, so the check's first forward and gradient pass with
    # the option back on are right only if those updates marked the images stale (fused tail, then the two-kernel tail)
    "idqn2_tc_forward_off_last": (Case(), [(2, 1, 1), (3, 0, 1)]),
    "idqn4_tc_forward_off_last": (Case(N=4, B=48, T=12), [(2, 1, 1), (3, 0, 1)]),
    "idqn2_tc_backward_off_last": (Case(), [(2, 1, 1), (4, 1, 0)]),               # W2^T image maintained by the Adam step alone, then read
    "idqn_shared_tc_backward_off_last": (Case(sharing=True, tu=0.05), [(1, 1, 1), (3, 1, 0)]),
    "vdn2_ends_on_hard_sync": (Case(mixer=1), [(3, 1, 1)]),
}


@pytest.mark.parametrize("case", list(IMAGE_CASES))
def test_images_kept_by_adam_equal_a_full_repack(case):
    """pack_param (the Adam step's per-parameter image update) is the function pack_weights_kernel uses, so this is bitwise: online and target
    forward and a tensor-core gradient pass give the same bits before and after params_changed() forces a repack of all three images."""
    c, phases = IMAGE_CASES[case]
    torch.manual_seed(5)
    m = _learner(c)
    _perturb_target(m)
    rng = np.random.default_rng(77)
    ts = _device_store(random_store(rng, c.cap, c.N, c.T, c.D, c.mixer != 0), c, m.device)
    first = 0
    for k, tcf, tcb in phases:
        _opt(b"tensor_core_forward", tcf); _opt(b"tensor_core_backward", tcb)
        m.update_n(ts, c.B, c.n_valid, SEED, first, k)
        first += k
    _opt(b"tensor_core_forward", True); _opt(b"tensor_core_backward", True)
    updates, last = _counters(m)
    assert updates == first
    if c.tu > 1:
        assert last == first // int(c.tu) * int(c.tu)
    obs = torch.tensor(rng.integers(-1, 12, size=(257, c.N, c.D)), dtype=torch.float32, device=m.device)
    idx = torch.tensor(policy_ref.replay_sample(SEED, first, c.B, c.n_valid), device=m.device)

    def outputs():
        q, tq = m.q_values(obs).clone(), m.q_values(obs, target=True).clone()
        m.update_grads(ts, idx)
        return dict(q=q.cpu(), target_q=tq.cpu(), grad=m.grad.cpu().clone())

    kept = outputs()
    m.params_changed()
    repacked = outputs()
    for k in kept:
        assert torch.equal(kept[k], repacked[k]), f"{k}: max abs difference {float((kept[k] - repacked[k]).abs().max()):.3e}"
    m.close()

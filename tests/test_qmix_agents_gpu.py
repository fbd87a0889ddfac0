"""GPU: QMIX over its whole agent range (1 to 8 agents) and at the mixing kernel's shared-memory limit (csrc/qmix.cuh, csrc/dqn.cu), against the
oracle (oracle/qmix_ref.py, tests/qmix_options_ref.py) run in float64: one update per shape with both weight-gradient forms of the mixer
(the single-read micro-tile kernel and the 32 x 32 tile kernel that MARL_QMIX_WGRAD_TILES=1 selects), unglued update chains, update_n and the
shapes the learner must refuse.

The shapes, from the layout arithmetic of qmix_layout / qm_smem_bytes / qmix_micro_tiles (mirrored by _layout below and checked against the
library's parameter count and refusal message):

  N   D    S    mixer (hl, E, He)   qmix_mix_kernel smem   micro-tiles (rounds of 512)   agents' training pass
  1   6    6    2, 64, 32           66.2 KB                217 (1)                       tensor cores
  5   18   90   2, 64, 32           210.7 KB               1065 (3)                      tensor cores
  5   21   105  2, 64, 32           223.9 KB (largest)     1161 (3)                      tensor cores
  6   24   144  1, 64, -            211.3 KB               2745 (6)                      tensor cores
  7   30   210  2, 32, 32           224.4 KB               1189 (3)                      tensor cores
  8   27   216  1, 32, -            166.0 KB               2469 (5)                      tensor cores
  8   32   256  2, 32, 16           208.5 KB               1013 (2)                      fused FP32 kernel (the tensor-core pass takes D < 32)
  5   22 / 23 with the default mixer need 228.3 / 232.7 KB and are refused, as are N = 9 and S > 256.
"""
import copy
import ctypes as C
import dataclasses
import json
import types

import numpy as np
import pytest
import torch

from oracle import learner_ref as lr
from oracle import policy_ref
from oracle import qmix_ref as qr
from tests import qmix_options_ref as qo
from tests.helpers import TIE, NearTie, assert_grad_close, random_store, redraw_on_near_tie, space, traj_store
from tests.test_qmix_options_gpu import _check_ret_ms, _close, _perturb_target, _state, _to_store

A = 6
SEED = 0x0A6E_5EED
WGRAD_TILES = "MARL_QMIX_WGRAD_TILES"
FORMS = ("micro", "tiles")   # qmix_wgrad2_kernel (default) / qmix_wgrad_kernel (MARL_QMIX_WGRAD_TILES=1)
BLOCK_TOL = 1e-5             # mixer gradient, per layer block, relative to the block's largest float64 element
SMEM_CAP = 227 * 1024


@dataclasses.dataclass(frozen=True)
class Case:
    N: int
    D: int
    hl: int = 2
    E: int = 64
    He: int = 32
    T: int = 8
    B: int = 16
    sharing: bool = False
    double_q: bool = True
    tu: float = 2.0
    standardise: bool = False

    @property
    def S(self):
        return self.N * self.D


def _layout(N, S, E, He, hl):
    """Python mirror of qmix_layout, qm_smem_bytes and qmix_micro_tiles (csrc/qmix.cuh): the mixer's parameter count, qmix_mix_kernel's dynamic
    shared memory (the resident image, without W1 when hl == 1, + 33-float rows of the tile's activations), the single-read weight-gradient
    kernel's micro-tiles (4 outputs x 8 inputs, bias = column I) and its shared memory (R record fields + the zero and the one field)."""
    lins = qo.mixer_shapes(N, S, E, He, hl)
    He = He if hl == 2 else 0
    n = sum(o * i + o for o, i in lins)
    res0 = N * E * S if hl == 1 else 0
    R = S + 4 * He + 4 * E + N * E + 1
    act_rows = S + 2 * He + 3 * E + N * E + N + 8 + 8 * N
    return dict(n=n, smem=(((n - res0 + 3) & ~3) + act_rows * 33) * 4, micro=sum(-(-o // 4) * (i // 8 + 1) for o, i in lins), wgrad2_smem=(R + 2) * 33 * 4)


def _layout_of(c):
    return _layout(c.N, c.S, c.E, c.He, c.hl)


def _hp(c):
    return lr.DqnHP(double_q=c.double_q, target_update_interval_or_tau=c.tu)


def _model(c, monkeypatch, form="micro"):
    """the handle reads MARL_QMIX_WGRAD_TILES once, in marl_dqn_qmix_init"""
    from codebase_b200.dqn import model as M

    if form == "tiles":
        monkeypatch.setenv(WGRAD_TILES, "1")
    else:
        monkeypatch.delenv(WGRAD_TILES, raising=False)
    hp = _hp(c)
    cfg = types.SimpleNamespace(optimizer="Adam", lr=hp.lr, gamma=hp.gamma, grad_clip=hp.grad_clip, double_q=c.double_q, target_update_interval_or_tau=c.tu,
                                standardise_returns=c.standardise)
    return M.QMixNetwork([space(shape=(c.D,))] * c.N, [space(n=A)] * c.N, cfg, [128, 128], c.sharing, False, True,
                         dict(embed_dim=c.E, hypernet_layers=c.hl, hypernet_embed=c.He), "cuda", max_batch=c.B, max_episode_length=c.T)


def _copy_params(src, dst):
    for k in ("theta", "theta_tgt", "mix", "mix_tgt"):
        getattr(dst, k).copy_(getattr(src, k))
    dst.params_changed()


def _oracle(c, m):
    """the oracle's state in float64, from the learner's float32 parameters"""
    f = lambda t: t.detach().cpu().double().clone()
    ret_ms = None
    if c.standardise:
        ret_ms = lr.RunningMeanStdRef((1,))
        ret_ms.mean, ret_ms.var = ret_ms.mean.double(), ret_ms.var.double()
    return qo.QmixOptState(f(m.theta), f(m.theta_tgt), f(m.mix), f(m.mix_tgt), [0] * c.N if c.sharing else list(range(c.N)), c.D, A,
                           embed_dim=c.E, hypernet_embed=c.He, hypernet_layers=c.hl, ret_ms=ret_ms)


def _f64(batch):
    return {k: v.double() if v.is_floating_point() else v for k, v in batch.items()}


def _margin(c, st, b, hp):
    if c.double_q:
        margin = lr.double_q_margin(lr.DqnState(st.theta, st.theta_tgt, st.agent_net, c.D, A), b, hp)
        if margin < TIE:
            raise NearTie(f"double-Q argmax margin {margin:.1e}")


def _block_ratios(c, got, want, other=None):
    """per layer block of the mixer (weights and biases of every Linear): max |got - want| / (BLOCK_TOL x the block's largest |want|); with
    `other`, the gap between got and other on the same scale"""
    split = lambda v: qo.split_mixer(torch.as_tensor(np.asarray(v, np.float64)), c.N, c.S, c.E, c.He, c.hl)
    names = [f"{k}.{p}" for k in qo.mixer_keys(c.hl) for p in ("weight", "bias")]
    out = {}
    for name, g, w, o in zip(names, split(got), split(want), split(want if other is None else other)):
        scale = max(float(w.abs().max()), 1e-30)
        out[name] = float((g - o).abs().max()) / (BLOCK_TOL * scale)
    return out


def _assert_blocks(c, got, want, what, other=None):
    """every block within its bar; returns (worst block, its fraction of the bar)"""
    ratios = _block_ratios(c, got, want, other)
    bad = {k: round(v, 2) for k, v in ratios.items() if not v <= 1.0}
    assert not bad, f"{what}: mixer gradient blocks over {BLOCK_TOL:g} x their largest element (fraction of the bar): {bad}"
    worst = max(ratios, key=ratios.get)
    return worst, ratios[worst]


def _check_update(c, m, st, st0, b, want, met, hp, what, per_block):
    """loss, clip norm, the agents' gradient and the mixer's of one update (per layer block against the float64 oracle, or -- after earlier
    updates, when the two states have drifted apart by Adam's sign-led first steps on near-zero gradients -- the whole-mixer bar of
    tests/test_qmix_options_gpu.py); then both parameter sets, both targets and the running statistics.  Returns the worst mixer block."""
    filled = float(b["filled"].sum())
    assert abs(float(met[0]) - want["loss"]) <= 1e-5 * max(1.0, abs(want["loss"])), f"loss, {what}: {float(met[0])} vs {want['loss']}"
    got_mix = m.mix_grad[: m.n_mix].cpu().numpy() / filled
    worst = None
    if per_block:
        worst = _assert_blocks(c, got_mix, want["mix_grad"].numpy(), what)
    else:
        _close(got_mix, want["mix_grad"].numpy(), 2e-5, f"mixer gradient, {what}")
    assert_grad_close(lr, st0, b, hp, m.grad[: m.n_params].cpu().numpy() / filled, want["grad"].numpy(), tol=2e-5, what=f"agents' gradient, {what}",
                      kink_risk=lambda: qo.qmix_kink_risk(st0, b, hp))
    assert abs(float(met[1]) - want["grad_norm"]) <= 2e-5 * max(1.0, want["grad_norm"]), f"clip norm, {what}: {float(met[1])} vs {want['grad_norm']}"
    for mine, theirs, name in ((m.theta, st.theta, "theta"), (m.mix, st.mix, "mixer"), (m.theta_tgt, st.theta_tgt, "target"), (m.mix_tgt, st.mix_tgt, "target mixer")):
        assert np.quantile(np.abs(mine.cpu().numpy() - theirs.numpy()), 0.999) < 2e-5, f"{name} after {what}"
    if c.standardise:
        _check_ret_ms(m, st, what)
    return worst


def _mixer_launches(m, ts, idx, tmp_path):
    """one update under torch.profiler: how many times the mixing kernel and each weight-gradient kernel of the mixer ran"""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        m.update_from_store(ts, idx)
        torch.cuda.synchronize()
    trace = tmp_path / "trace.json"
    prof.export_chrome_trace(str(trace))
    names = [e.get("name", "") for e in json.loads(trace.read_text())["traceEvents"] if e.get("cat") == "kernel"]
    return {k: sum(k in s for s in names) for k in ("qmix_mix_kernel", "qmix_wgrad_kernel", "qmix_wgrad2_kernel")}


# ---- the shapes' edges (no GPU: the layout mirror against the library) ---------------------------------------------------------------------------
SHAPES = {
    "n1_d6": Case(N=1, D=6, T=8, B=16),
    "n5_d18_shared_single_q": Case(N=5, D=18, T=10, B=16, sharing=True, double_q=False),
    "n5_d21": Case(N=5, D=21, T=12, B=24),
    "n6_d24_h1_shared": Case(N=6, D=24, hl=1, T=8, B=16, sharing=True, tu=0.05),
    "n7_d30_e32_single_q": Case(N=7, D=30, E=32, T=6, B=32, double_q=False),
    "n8_d27_h1_e32": Case(N=8, D=27, hl=1, E=32, T=10, B=16),
    "n8_d32_e32_he16_shared": Case(N=8, D=32, E=32, He=16, T=7, B=12, sharing=True),
}


def test_shapes_reach_the_edges_they_test():
    """the mirror's parameter count is the library's; the cases hold what they are there for: N = 1..8, hl 1 and 2, the largest default mixer
    (D = 21 at N = 5 fits, D = 22 does not), five and six rounds of micro-tiles, S = 256, and every case on the single-read form by default"""
    from codebase_b200 import _native as nat

    for c in SHAPES.values():
        n = C.c_int64()
        nat.check(nat.lib().marl_debug_qmix_coverage_layers(C.c_int32(c.N), C.c_int32(c.S), C.c_int32(c.E), C.c_int32(c.hl), C.c_int32(c.He), None,
                                                            C.c_int64(0), C.byref(n)), "marl_debug_qmix_coverage_layers")
        L = _layout_of(c)
        assert L["n"] == n.value == qo.mixer_size(c.N, c.S, c.E, c.He, c.hl), c
        assert L["smem"] <= SMEM_CAP and L["wgrad2_smem"] <= 110 * 1024, c
    assert {c.N for c in SHAPES.values()} == {1, 5, 6, 7, 8} and {c.hl for c in SHAPES.values()} == {1, 2}
    big = _layout_of(SHAPES["n5_d21"])
    assert SMEM_CAP - 4 * 1024 < big["smem"] <= SMEM_CAP and _layout(5, 110, 64, 32, 2)["smem"] > SMEM_CAP
    assert -(-_layout_of(SHAPES["n8_d27_h1_e32"])["micro"] // 512) == 5 and -(-_layout_of(SHAPES["n6_d24_h1_shared"])["micro"] // 512) == 6
    assert SHAPES["n8_d32_e32_he16_shared"].S == 256


# ---- 1 + 2. one update per shape, both weight-gradient forms -------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("name", list(SHAPES))
@redraw_on_near_tie
def test_one_update_matches_the_float64_oracle(name, form, monkeypatch, tmp_path):
    """ragged episodes through marl_dqn_update: loss, clip norm, the agents' gradient, the mixer's gradient per layer block, the parameters after the
    step.  A second handle of the same form repeats the update bit for bit, and the profiler shows the form's kernel ran (micro-tiles: once per
    round of 512)."""
    c = SHAPES[name]
    hp = _hp(c)
    m = _model(c, monkeypatch, form)
    _perturb_target(m)
    twin = _model(c, monkeypatch, form)
    _copy_params(m, twin)
    st = _oracle(c, m)
    batch = qr.random_batch(c.N, c.T, c.B, c.D, A, seed=100 * c.N + c.B, ragged=True)
    b64 = _f64(batch)
    _margin(c, st, b64, hp)
    st0 = copy.deepcopy(st)
    want = qo.qmix_update(st, b64, hp)
    ts = _to_store(batch, m.device)
    idx = torch.arange(c.B, dtype=torch.int32, device=m.device)
    met = m.update_from_store(ts, idx).cpu()
    launches = _mixer_launches(twin, ts, idx, tmp_path)
    rounds = -(-_layout_of(c)["micro"] // 512)
    expected = dict(qmix_mix_kernel=1, qmix_wgrad_kernel=0, qmix_wgrad2_kernel=rounds) if form == "micro" else \
        dict(qmix_mix_kernel=1, qmix_wgrad_kernel=1, qmix_wgrad2_kernel=0)
    assert launches == expected, f"kernel launches of one update: {launches}"
    mine, again = _state(m), _state(twin)
    for k in mine:
        assert torch.equal(mine[k], again[k]), f"{k} differs between two handles of the {form} form"
    blk, ratio = _check_update(c, m, st, st0, b64, want, met, hp, f"{name}, {form} form", per_block=True)
    print(f"{name} [{form}]: worst mixer block {blk} at {ratio:.3f} of the {BLOCK_TOL:g} bar")
    m.close(); twin.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SHAPES))
@redraw_on_near_tie
def test_weight_gradient_forms_agree(name, monkeypatch):
    """the same update on one handle of each form: the mixing kernel is shared, so the loss and the agents' gradient are identical; the two mixer
    gradients agree per layer block to the float64 bar, and each meets that bar against the oracle"""
    c = SHAPES[name]
    hp = _hp(c)
    a = _model(c, monkeypatch, "micro")
    _perturb_target(a)
    b = _model(c, monkeypatch, "tiles")
    _copy_params(a, b)
    st = _oracle(c, a)
    batch = qr.random_batch(c.N, c.T, c.B, c.D, A, seed=7 * c.N + c.B + 1, ragged=True)
    b64 = _f64(batch)
    _margin(c, st, b64, hp)
    want = qo.qmix_update(st, b64, hp)["mix_grad"].numpy()
    ts = _to_store(batch, a.device)
    idx = torch.arange(c.B, dtype=torch.int32, device=a.device)
    met_a, met_b = a.update_from_store(ts, idx).cpu(), b.update_from_store(ts, idx).cpu()
    assert torch.equal(met_a[:2], met_b[:2]) and torch.equal(a.grad.cpu(), b.grad.cpu()), "loss / agents' gradient differ between the forms"
    filled = float(batch["filled"].sum())
    ga, gb = a.mix_grad[: a.n_mix].cpu().numpy() / filled, b.mix_grad[: b.n_mix].cpu().numpy() / filled
    assert np.array_equal(a.mix_grad[a.n_mix:].cpu().numpy(), b.mix_grad[b.n_mix:].cpu().numpy()), "loss statistics of the mixer"
    (_, ra), (_, rb) = _assert_blocks(c, ga, want, "micro form"), _assert_blocks(c, gb, want, "tile form")
    blk, rx = _assert_blocks(c, ga, want, "micro vs tile form", other=gb)
    print(f"{name}: mixer gradient at {ra:.3f} (micro), {rb:.3f} (tiles), micro vs tiles {rx:.3f} ({blk}) of the {BLOCK_TOL:g} bar")
    a.close(); b.close()


# ---- 3. unglued update chains at the top of the range ------------------------------------------------------------------------------------------
CHAINS = {
    "n8_d27_h1_e32_std_polyak": Case(N=8, D=27, hl=1, E=32, T=10, B=16, standardise=True, tu=0.05),
    "n5_d21_hard": Case(N=5, D=21, T=12, B=16, tu=2.0),
    "n1_d6_h1_single_q": Case(N=1, D=6, hl=1, T=8, B=16, double_q=False, tu=3.0),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CHAINS))
@redraw_on_near_tie
def test_unglued_chain_matches_the_float64_oracle(name, monkeypatch):
    """three updates through marl_dqn_update on ragged episodes, never re-synchronised with the oracle, which takes the same batches in step (the
    hard-sync chain copies both targets at update 2, the Polyak chain moves them every update); the running statistics after each update"""
    c = CHAINS[name]
    hp = _hp(c)
    m = _model(c, monkeypatch)
    _perturb_target(m)
    st = _oracle(c, m)
    idx = torch.arange(c.B, dtype=torch.int32, device=m.device)
    for u in range(3):
        batch = qr.random_batch(c.N, c.T, c.B, c.D, A, seed=1000 * u + 10 * c.N + c.B, ragged=True)
        b64 = _f64(batch)
        _margin(c, st, b64, hp)
        st0 = copy.deepcopy(st)
        want = qo.qmix_update(st, b64, hp)
        met = m.update_from_store(_to_store(batch, m.device), idx).cpu()
        _check_update(c, m, st, st0, b64, want, met, hp, f"update {u}", per_block=u == 0)
    assert m.updates == 3
    m.close()


# ---- 4. update_n at N >= 5: the loop it replaces, bit for bit, and the oracle --------------------------------------------------------------------
UPDATE_N = {
    "n5_d18": Case(N=5, D=18, T=10, B=16, tu=3.0),
    "n8_d27_h1_e32_std": Case(N=8, D=27, hl=1, E=32, T=10, B=16, standardise=True, tu=0.05),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(UPDATE_N))
@redraw_on_near_tie
def test_update_n_is_the_loop_it_replaces_and_tracks_the_oracle(name, monkeypatch):
    from codebase_b200 import _native as nat
    from codebase_b200.lbf import TrajStore

    c, K, cap = UPDATE_N[name], 4, 48
    hp = _hp(c)
    a = _model(c, monkeypatch)
    _perturb_target(a)
    b = _model(c, monkeypatch)
    _copy_params(a, b)
    st = _oracle(c, a)
    store = random_store(np.random.default_rng(c.N * 100 + c.B), cap, c.N, c.T, c.D, True, A=A)
    ts = TrajStore(cap, c.N, c.T, c.D, a.device)
    for k in ("obs", "act", "rew", "done", "filled"):
        getattr(ts, k).copy_(torch.as_tensor(store[k]))
    a.update_n(ts, c.B, cap, SEED, 0, K)
    idx = torch.zeros(c.B, dtype=torch.int32, device=b.device)
    for u in range(K):
        nat.check(nat.lib().marl_replay_sample(C.c_uint64(SEED), C.c_uint64(u), C.c_int32(c.B), C.c_int32(cap), nat.ptr(idx), nat.stream_ptr()), "marl_replay_sample")
        ids = policy_ref.replay_sample(SEED, u, c.B, cap)
        assert np.array_equal(idx.cpu().numpy(), ids), f"replay indices of update {u}"
        b64 = _f64(lr.batch_from_store(store, ids))
        _margin(c, st, b64, hp)
        st0 = copy.deepcopy(st)
        want = qo.qmix_update(st, b64, hp)
        met = b.update_from_store(ts, idx).cpu()
        _check_update(c, b, st, st0, b64, want, met, hp, f"update {u}", per_block=u == 0)
    got, ref = _state(a), _state(b)
    assert got.keys() == ref.keys()
    for k in ref:
        assert torch.equal(got[k], ref[k]), f"{k}: max abs difference {float((got[k].double() - ref[k].double()).abs().max()):.3e}"
    assert a.updates == b.updates == K
    a.close(); b.close()


# ---- 5. the acceptance edge ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_largest_default_mixer_is_created_and_trains(monkeypatch):
    """N = 5, D = 21 with the default mixer needs 223.9 KB of qmix_mix_kernel's 227 KB: created, and trained by update_n on a replay store"""
    c = SHAPES["n5_d21"]
    m = _model(c, monkeypatch)
    assert m.n_mix == qo.mixer_size(c.N, c.S, c.E, c.He, c.hl)
    store = random_store(np.random.default_rng(21), 64, c.N, c.T, c.D, True, A=A)
    theta0, mix0 = m.theta.clone(), m.mix.clone()
    met = m.update_n(traj_store(store, m.device), c.B, 64, SEED, 0, 6).cpu()
    assert m.updates == 6 and np.isfinite(float(met[0])) and np.isfinite(float(met[1])) and float(met[1]) > 0
    assert bool(torch.isfinite(m.theta).all()) and bool(torch.isfinite(m.mix).all())
    assert float((m.theta - theta0).abs().max()) > 0 and float((m.mix - mix0).abs().max()) > 0
    m.close()


REFUSED = {
    "n5_d22_default": (Case(N=5, D=22), "native"),
    "n5_d23_default": (Case(N=5, D=23), "native"),
    "n9": (Case(N=9, D=6), "n_agents must be 1..8"),
    "s264": (Case(N=8, D=33, E=32, He=16), "state_dim must be 1..256"),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(REFUSED))
def test_refused_shapes_fail_cleanly_and_leave_the_device_usable(name, monkeypatch):
    """a mixer that does not fit qmix_mix_kernel's shared memory is refused by marl_dqn_qmix_init (MARL_EINVAL, the byte count in the message);
    N = 9 and S > 256 are refused in Python before any native call.  Either way the refusal comes before any mixer kernel is launched: the device
    has no pending error and a learner created next trains"""
    from codebase_b200 import _native as nat

    c, why = REFUSED[name]
    if why == "native":
        need = _layout_of(c)["smem"]
        assert need > SMEM_CAP
        with pytest.raises(nat.NativeError, match=rf"marl_dqn_qmix_init failed \(rc=-1\): .*\({need} bytes\) do not fit shared memory"):
            _model(c, monkeypatch)
    else:
        with pytest.raises(NotImplementedError, match=why):
            _model(c, monkeypatch)
    torch.cuda.synchronize()
    ok = Case(N=2, D=9, B=8, T=6)
    m = _model(ok, monkeypatch)
    met = m.update_from_store(_to_store(qr.random_batch(ok.N, ok.T, ok.B, ok.D, A, seed=3), m.device), torch.arange(ok.B, dtype=torch.int32, device=m.device)).cpu()
    assert np.isfinite(float(met[0])) and m.updates == 1
    m.close()

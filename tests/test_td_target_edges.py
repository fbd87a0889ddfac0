"""The DQN family's TD(λ) targets on the CPU: what tests/test_td_target_edges_gpu.py relies on.

- The split mirror (tests/returns_ref.py): every GPU case reaches the window, lane, block and standardisation boundaries it is listed for, and
  together the cases reach every one of them.
- The per-row bar |got - want| <= τ S_t (returns_ref.td_tau), with S_t the TD(λ) target's no-cancellation scale cut at the first unfilled row: a plain float32
  recursion in td_lambda_kernel's arithmetic passes it with at least 8x margin, and each plausible defect of the scan (a dropped carry, f_{t+1}
  read as f_t, a lane's incoming G from the wrong lane, a shifted window edge, a cut ignored on a window's last step) fails it by 100x or more.
Run with -s to see each case's boundaries, the float32 recursion's margin and each defect's factor over the bar."""
import numpy as np
import pytest
import torch

from tests import returns_ref as rr
from tests import td_lambda_ref as tl

# what each case of the GPU sweep is there for (checked against the mirror, not derived from it)
CLAIMS = {
    1: {"windows=1", "T%256=1", "CB<8"},
    7: {"windows=1", "T%256=7", "CB%8=1", "CBT%256=255", "partial last block", "ret_ms cols"},
    9: {"T%256=9", "CB%8=7", "cut at a lane edge", "restart at a lane edge", "done at a lane edge"},
    255: {"T%256=255", "CB%8=0", "cut at a lane edge", "restart at a lane edge"},
    256: {"T%256=0", "CBT%256=0", "CB%8=1", "done at a lane edge"},
    257: {"windows=2", "T%256=1", "CB%8=7", "CBT%256=255", "cut at w0-1", "cut at w0", "restart at w0-1", "restart at w0", "done at w0",
          "ret_ms cols"},
    263: {"windows=2", "T%256=7", "CB%8=1", "cut at w0+1", "restart at w0+1", "done at w0-1"},
    264: {"windows=2", "T%256=8", "CB%8=0", "cut at w0", "restart at w0", "done at w0+1"},
    265: {"windows=2", "T%256=9", "CB%8=1", "CBT%256=1", "cut at w0-1", "restart at w0-1", "done at w0"},
    511: {"windows=2", "T%256=255", "CB%8=7", "cut at a lane edge", "done at w0"},
    512: {"windows=2", "T%256=0", "CB%8=7", "CBT%256=0", "restart at w0"},
    769: {"windows=4", "T%256=1", "CB%8=0", "cut at w0", "done at w0-1"},
    1024: {"windows=4", "T%256=0", "CB%8=1", "CBT%256=0", "restart at w0+1", "ret_ms cols"},
    1025: {"windows=5", "T%256=1", "CB%8=1", "cut at w0-1", "cut at w0", "cut at w0+1", "restart at w0", "done at w0+1"},
}
NEEDED = ({f"T%256={m}" for m in (1, 7, 8, 9, 255, 0)} | {f"windows={w}" for w in range(1, 6)} - {"windows=3"}
          | {"CB%8=0", "CB%8=1", "CB%8=7", "CB<8", "CBT%256=255", "CBT%256=0", "CBT%256=1", "partial last block", "ret_ms cols", "ret_ms grid"}
          | {f"{e} at {w}" for e in ("cut", "restart", "done") for w in ("w0-1", "w0", "w0+1", "a lane edge")})


@pytest.mark.parametrize("T,kind,N,cb8,cbt", rr.TD_CASES)
def test_every_gpu_case_reaches_its_boundaries(T, kind, N, cb8, cbt):
    C, B = rr.td_case(T, kind, N, cb8, cbt)
    got = rr.td_reaches(T, kind, N, B, standardise=True)
    print(f"T={T} {kind} C={C} B={B}: windows {rr.windows(T)}: {sorted(got)}")
    assert B >= min(len(rr.td_episodes(T)), 3)
    missing = CLAIMS[T] - got
    assert not missing, missing


def test_the_cases_cover_every_boundary():
    assert {c[0] for c in rr.TD_CASES} == set(CLAIMS)
    assert {c[1] for c in rr.TD_CASES} == {"idqn", "vdn", "qmix"}
    union = set().union(*(rr.td_reaches(c[0], c[1], c[2], rr.td_case(*c)[1], standardise=True) for c in rr.TD_CASES))
    assert NEEDED <= union, NEEDED - union


def test_batch_places_its_events():
    """the scripted episodes of td_batch: a cut leaves x unfilled, a done ends at x, a stale tail restarts at x after one unfilled row"""
    T = 264
    s = rr.td_batch(np.random.default_rng(0), T, 2, len(rr.td_episodes(T)))
    for e, (kind, x) in enumerate(rr.td_episodes(T)):
        f, d = s["filled"][e], s["done"][e]
        if kind == "cut":
            assert f[:x].all() and not f[x:].any() and not d.any()
        elif kind == "done":
            assert f[:x].all() and not f[x:].any() and d[x] == 1 and d.sum() == 1
        elif kind == "stale":
            assert f[: x - 1].all() and f[x - 1] == 0 and f[x:].all()
        else:
            assert f.all() and not d[:T].any()


def test_ret_ms_path():
    assert rr.ret_ms_path("vdn", 2, 64, 25) == "grid" and rr.ret_ms_path("vdn", 2, 65, 25) == "cols"
    assert rr.ret_ms_path("qmix", 2, 128, 1024) == "cols" and rr.ret_ms_path("qmix", 2, 128, 1025) == "grid"
    assert rr.ret_ms_path("idqn", 32, 128, 8) == "grid"


def test_scale_is_cut_at_the_first_unfilled_row():
    """S_t sees nothing after the first unfilled row, and bounds |G_t| for any rewards and bootstrap values"""
    rng = np.random.default_rng(1)
    T = 40
    r, v = rng.standard_normal((T, 6)), rng.standard_normal((T, 6))
    d = (rng.random((T + 1, 6)) < 0.1).astype(np.float64)
    f = np.ones((T, 6)); f[20:, :3] = 0; f[25:, 3:] = 1
    S = rr.td_lambda_scale(r, d, f, v, 0.9, 0.99)
    G = tl.lambda_targets(*(torch.tensor(x) for x in (r, d, f, v)), 0.9, 0.99).numpy()
    assert (np.abs(G) <= S * (1 + 1e-12)).all()
    r2 = r.copy(); r2[20:, :3] += 100.0
    assert np.array_equal(rr.td_lambda_scale(r2, d, f, v, 0.9, 0.99)[:20, :3], S[:20, :3])


# ---- the per-row bar -------------------------------------------------------------------------------------------------------------------------------
_DATA = {}


def _case_data(T, kind, N, cb8, cbt):
    """a GPU case's rewards, dones and filled flags with stand-in bootstrap values, and {(γ, λ): (want, S)}, computed once"""
    if T not in _DATA:
        C, B = rr.td_case(T, kind, N, cb8, cbt)
        s = rr.td_batch(np.random.default_rng(T), T, N, B)
        rew, done, filled = rr.td_sequences(s, C)
        boot = np.random.default_rng(T + 1).standard_normal(rew.shape).astype(np.float32).astype(np.float64)
        want = {}
        for g in rr.GAMMAS:
            for lam in rr.LAMBDAS:
                l32, g32 = float(np.float32(lam)), float(np.float32(g))
                w = tl.lambda_targets(*(torch.tensor(np.ascontiguousarray(x)) for x in (rew, done, filled, boot)), l32, g32).numpy()
                want[(g, lam)] = (w, rr.td_lambda_scale(rew, done, filled, boot, l32, g32))
        _DATA[T] = ((rew, done, filled, boot, s), want)
    return _DATA[T]


@pytest.mark.parametrize("T,kind,N,cb8,cbt", rr.TD_CASES)
def test_float32_recursion_passes_the_bar_with_margin(T, kind, N, cb8, cbt):
    (rew, done, filled, boot, _), want = _case_data(T, kind, N, cb8, cbt)
    for (gamma, lam), (w, S) in want.items():
        got = rr.td_f32_recursion(rew, done, filled, boot, lam, gamma)
        ratio = rr.worst(got, w, S, rr.td_tau(T, gamma, lam))
        print(f"T={T} γ={gamma} λ={lam}: τ = {rr.td_tau(T, gamma, lam):.2e}, float32 recursion at {ratio:.3f} of the bar ({1 / max(ratio, 1e-9):.0f}x margin)")
        assert ratio <= 1 / 8, (gamma, lam, ratio)


MUTATIONS = ("carry between windows dropped", "f_{t+1} read as f_t", "a lane's incoming G from two lanes over", "window edge shifted by one",
             "cut ignored on a window's last step")


@pytest.mark.parametrize("name", MUTATIONS)
def test_defects_of_the_scan_fail_the_bar(name):
    """each defect fails the bar by 100x or more at every λ > 0 of every case it applies to (at λ = 0 the scan has no chain to get wrong)"""
    applied = []
    for case in rr.TD_CASES:
        T = case[0]
        (rew, done, filled, boot, s), want = _case_data(*case)
        cut_rows = {int(t) for t in range(1, T) if ((filled[t - 1] > 0) & (filled[t] == 0)).any()}
        kw = rr.td_mutations(T, cut_rows).get(name)
        if kw is None:
            continue
        worst = np.inf
        for (gamma, lam), (w, S) in want.items():
            if lam == 0.0:
                continue
            factor = rr.worst(rr.td_f32_recursion(rew, done, filled, boot, lam, gamma, **kw), w, S, rr.td_tau(T, gamma, lam))
            worst = min(worst, factor)
        print(f"{name}: T={T}: at least {worst:.0f}x the bar")
        assert worst >= 100, (name, T, worst)
        applied.append(T)
    assert len(applied) >= 2 and max(applied) >= 769, applied

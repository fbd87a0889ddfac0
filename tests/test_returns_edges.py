"""The actor-critic return pass on the CPU: what tests/test_returns_edges_gpu.py relies on.

- The split mirror: every GPU λ case reaches the window, lane and block boundaries it is listed for.
- The streamed float64 mixture of tests/gae_ref.py: equal to the stacked one at the old sizes, and to the hand-written recursion at several windows.
- The per-row bar |got - want| <= τ S_t: a plain float32 recursion passes it with room to spare on every long case, and each plausible defect of the
  split (a dropped or misplaced carry, a shifted edge, an ignored done, a chunk replayed from the wrong step) fails it by two orders of magnitude.
- The standardisation bar: float32 batch moments miss the variance of the offset case (mean 50, spread 0.01) by far more than it allows, the
  kernel's FP64 moments with its float32 running update stay inside it.
Run with -s to see each case's boundaries, the float32 recursion's margin and each defect's factor over the bar."""
import numpy as np
import pytest
import torch

from oracle import learner_ref as lr
from tests import gae_ref as gr
from tests import returns_ref as rr

# what each λ case of the GPU sweep is there for (checked against the mirror, not derived from it)
CLAIMS = {
    (7, 1): {"windows=1", "partial lane chunk", "untruncated full-length episode", "block class"},
    (8, 3): {"windows=1", "full lane chunks", "block class"},
    (9, 1): {"windows=1", "one-step lane chunk", "done at a chunk edge", "block class"},
    (15, 2): {"partial lane chunk", "done at a chunk edge", "block class"},
    (16, 3): {"full lane chunks", "done at a chunk edge", "block class"},
    (17, 1): {"one-step lane chunk", "done at a chunk edge", "block class"},
    (255, 1): {"windows=1", "partial lane chunk", "done at a chunk edge", "block class"},
    (256, 2): {"windows=1", "full last window", "full lane chunks", "done at a chunk edge", "block class"},
    (257, 3): {"windows=2", "one-step window", "one-step lane chunk", "done at w0 - 1", "done at w0", "done at w0 + 1", "block class"},
    (257, 32): {"windows=2", "one-step window", "N = 32", "done at w0 - 1", "done at w0", "block class"},
    (511, 1): {"windows=2", "partial lane chunk", "done at w0 - 1", "done at w0", "done at w0 + 1", "done at a chunk edge", "block class"},
    (512, 1): {"windows=2", "full last window", "done at w0 - 1", "done at w0", "done at w0 + 1", "block class"},
    (513, 2): {">= 3 windows", "windows=3", "one-step window", "done at w0 - 1", "done at w0", "done at w0 + 1", "block class"},
    (769, 1): {">= 3 windows", "windows=4", "one-step window", "done at w0 + 1", "block class"},
    (1025, 1): {">= 3 windows", "windows=5", "one-step window", "done at w0 - 1", "done at w0", "done at w0 + 1", "done at a chunk edge",
                "untruncated full-length episode", "block class"},
}
NEEDED = {"one-step window", "full last window", ">= 3 windows", "done at w0 - 1", "done at w0", "done at w0 + 1", "done at a chunk edge",
          "untruncated full-length episode", "N = 32", "NP%8=1", "NP%8=0", "partial lane chunk", "one-step lane chunk", "full lane chunks"}


def test_mirror_of_the_split():
    assert rr.windows(1) == [(0, 1)]
    assert rr.windows(256) == [(0, 256)]
    assert rr.windows(257) == [(256, 1), (0, 256)]
    assert rr.windows(1025) == [(1024, 1), (768, 256), (512, 256), (256, 256), (0, 256)]
    assert rr.lanes(256)[31] == (248, 256) and rr.lanes(9)[1] == (8, 9) and rr.lanes(9)[2][1] <= rr.lanes(9)[2][0]
    for T in (1, 7, 255, 256, 257, 1025):   # the windows and lanes tile [0, T) once
        steps = [w0 + t for w0, length in rr.windows(T) for lo, hi in rr.lanes(length) for t in range(lo, hi)]
        assert sorted(steps) == list(range(T))


@pytest.mark.parametrize("T,N,block", rr.LAMBDA_CASES)
def test_every_gpu_case_reaches_its_boundaries(T, N, block):
    P = rr.case_P(T, N, block)
    got = rr.reaches(T, N, P, block)
    print(f"T={T} N={N} P={P}: windows {rr.windows(T)}, dones at {rr.done_at(T)}: {sorted(got)}")
    missing = CLAIMS[(T, N)] - got
    assert not missing, missing


def test_the_cases_cover_every_boundary():
    assert {(T, N) for T, N, _ in rr.LAMBDA_CASES} == set(CLAIMS)
    assert {T for T, _, _ in rr.LAMBDA_CASES} == set(rr.LAMBDA_TS)
    union = set().union(*(rr.reaches(T, N, rr.case_P(T, N, b), b) for T, N, b in rr.LAMBDA_CASES))
    assert NEEDED <= union, NEEDED - union


# ---- the streamed mixture --------------------------------------------------------------------------------------------------------------------------
def _sequences(rng, T, B=3, N=2):
    rew = rng.standard_normal((T, B, N))
    done = np.zeros((T + 1, B, N))
    for b in range(B):
        end = int(rng.integers(1, T + 1))
        done[end, b] = 1.0
    return rew, done, rng.standard_normal((T + 1, B, N))


@pytest.mark.parametrize("T", [1, 2, 7, 33])
def test_streamed_mixture_equals_the_stacked_one(T):
    rew, done, v = _sequences(np.random.default_rng(T), T)
    for lam in (0.0, 0.3, 0.95, 1.0):
        G = gr.nstep_all(rew, done, v, 0.99)
        stacked = lam ** (T - 1) * G[T - 1] + sum((1.0 - lam) * lam ** (n - 1) * G[n - 1] for n in range(1, T))
        np.testing.assert_allclose(gr.lambda_returns(rew, done, v, lam, 0.99), stacked, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("T", [257, 513, 1025])
@pytest.mark.parametrize("gamma", [0.99, 0.999])
def test_mixture_equals_the_recursion_at_length(T, gamma):
    rew, done, v = _sequences(np.random.default_rng(T), T)
    for lam in (0.0, 0.5, 0.95, 1.0):
        np.testing.assert_allclose(gr.lambda_returns(rew, done, v, lam, gamma), gr.recursion(rew, done, v, lam, gamma), rtol=1e-12, atol=1e-12)


# ---- the per-row bar -------------------------------------------------------------------------------------------------------------------------------
def _case_data(T, N, block):
    """a GPU case's rewards and dones with stand-in target values (the critic's are only known on the device), float32 inputs"""
    P = rr.case_P(T, N, block)
    s = rr.lambda_batch(np.random.default_rng(T * 7 + N), T, N, P)
    rew, done, _ = rr.sequences(s)
    v = np.random.default_rng(T).standard_normal(done.shape).astype(np.float32).astype(np.float64)
    return rew, done, v, s


def _want(rew, done, v, lam, gamma):
    l32, g32 = float(np.float32(lam)), float(np.float32(gamma))
    return gr.lambda_returns(rew, done, v, l32, g32), rr.lambda_scale(rew, done, v, l32, g32)


LONG = [c for c in rr.LAMBDA_CASES if c[0] >= 255]
_MIXTURES = {}


def _mixtures(T, N, block):
    """(data, {(γ, λ): (want, S)}) of a case, computed once for the two tests below"""
    if (T, N) not in _MIXTURES:
        rew, done, v, s = _case_data(T, N, block)
        _MIXTURES[(T, N)] = ((rew, done, v, s), {(g, lam): _want(rew, done, v, lam, g) for g in rr.GAMMAS for lam in rr.LAMBDAS})
    return _MIXTURES[(T, N)]


@pytest.mark.parametrize("T,N,block", LONG)
def test_float32_recursion_passes_the_bar_with_margin(T, N, block):
    (rew, done, v, _), want = _mixtures(T, N, block)
    for (gamma, lam), (w, S) in want.items():
        got = rr.f32_recursion(rew, done, v, lam, gamma)
        ratio = rr.worst(got, w, S, rr.tau(T, gamma, lam))
        print(f"T={T} N={N} γ={gamma} λ={lam}: τ = {rr.tau(T, gamma, lam):.2e}, float32 recursion at {ratio:.3f} of the bar "
              f"({1 / ratio:.0f}x margin)")
        assert ratio <= 0.25, (gamma, lam, ratio)


@pytest.mark.parametrize("T,N,block", rr.LAMBDA_CASES)
def test_defects_of_the_split_fail_the_bar(T, N, block):
    (rew, done, v, s), want = _mixtures(T, N, block)
    done_rows = {int(i) for i in np.flatnonzero(s["done"].any(axis=0))}
    muts = rr.mutations(T, done_rows)
    for (gamma, lam), (w, S) in want.items():
        cv, cr = rr.coefs(lam, gamma)
        for name, kw in muts.items():
            if ("ignore_done_at" in kw and cv == 0) or ("next_of" in kw and cr == 0):
                continue   # the defect changes nothing here: no bootstrap (λ = 1), no carry (λ = 0)
            factor = rr.worst(rr.f32_recursion(rew, done, v, lam, gamma, **kw), w, S, rr.tau(T, gamma, lam))
            print(f"T={T} N={N} γ={gamma} λ={lam}: {name}: {factor:.0f}x the bar")
            assert factor >= 100, (name, gamma, lam, factor)


# ---- the standardisation bar -------------------------------------------------------------------------------------------------------------------
OFFSET_N = 16385   # P·T of the GPU offset case: one return past ret_moments_kernel's grid stride


def _offset_returns(rng, n=OFFSET_N):
    return (50.0 + 0.01 * rng.standard_normal(n)).astype(np.float32)


def test_float32_moments_miss_the_offset_variance():
    """the batch variance of returns with mean 50 and spread 0.01 from float32 sums (what an FP32 ret_moments_kernel would do) is off by far more
    than the 1e-6 relative bar; from FP64 sums it is inside it"""
    x = _offset_returns(np.random.default_rng(0))
    want = float(np.var(x.astype(np.float64), ddof=1))
    n = x.size

    def one_pass(dtype):
        s1, s2 = np.zeros((), dtype), np.zeros((), dtype)
        for chunk in x.astype(dtype).reshape(-1, 5):   # sequential partial sums, as one thread's strided loop then the block tree
            s1 = dtype(s1 + chunk.sum(dtype=dtype)); s2 = dtype(s2 + (chunk * chunk).sum(dtype=dtype))
        m = s1 / dtype(n)
        return float((s2 - dtype(n) * m * m) / dtype(n - 1))

    err32, err64 = abs(one_pass(np.float32) - want) / want, abs(one_pass(np.float64) - want) / want
    print(f"offset case: float32 moments miss the batch variance by {err32:.2e} relative, float64 by {err64:.2e} (bar 1e-6)")
    assert err32 >= 1e3 * 1e-6 and err64 <= 1e-8


def _device_update(mean, var, count, x):
    """csrc/retms.cuh's step: FP64 batch moments, then RunningMeanStd.update_from_moments in float32 operation by operation"""
    f = np.float32
    n = x.shape[0]
    s1, s2 = x.astype(np.float64).sum(0), (x.astype(np.float64) ** 2).sum(0)
    bm = s1 / n
    bv = (s2 - n * bm * bm) / (n - 1) if n > 1 else np.zeros_like(bm)
    bm32, bv32, bc = bm.astype(f), bv.astype(f), f(n)
    cnt, tot = f(count), f(count + n)
    delta = bm32 - mean
    new_mean = mean + (delta * bc) / tot
    m2 = (var * cnt + bv32 * bc) + ((delta * delta) * cnt * bc) / tot
    return new_mean.astype(f), (m2 / tot).astype(f), count + n


@pytest.mark.parametrize("offset", [0.0, 50.0])
def test_device_statistics_stay_inside_the_bar(offset):
    """three updates of the device's running statistics (FP64 moments, float32 update) against the float64 StatsRef inside its bar, at returns
    of mean 0 and spread 1 and at the offset case (mean 50, spread 0.01, a batch mean that moves by 1e-3 between updates); FP32 moments miss it
    by a factor of 1000 or more"""
    rng = np.random.default_rng(int(offset) + 1)
    ref = rr.StatsRef(4)
    mean, var, count = np.zeros(4, np.float32), np.ones(4, np.float32), 1e-4
    for u in range(3):
        x = (offset + (0.01 if offset else 1.0) * rng.standard_normal((OFFSET_N, 4)) + 0.001 * rng.standard_normal(4)).astype(np.float32)
        mean, var, count = _device_update(mean, var, count, x)
        ref.update(x)
        em = np.abs(mean - ref.mean) / np.abs(ref.mean)
        ev = np.abs(var - ref.var) / ref.var_bar
        print(f"offset {offset} update {u}: running mean off by {em.max():.1e} relative, var at {ev.max():.2f} of its bar "
              f"({(ref.var_bar / ref.var).max():.1e} relative)")
        assert em.max() <= 1e-6 and ev.max() <= 1.0 and count == ref.count
    if offset:
        bad = _fp32_moments_update(x[:, 0])
        first = rr.StatsRef(1)
        first.update(x[:, :1])
        factor = float(abs(bad - first.var[0]) / first.var_bar[0])
        print(f"offset case: FP32 moments put the first update's running var at {factor:.0f}x its bar")
        assert factor >= 1000


def _fp32_moments_update(x):
    """the first update's running var with the batch moments summed in float32"""
    f = np.float32
    n = x.size
    s1, s2 = np.sum(x, dtype=f), np.sum(x * x, dtype=f)
    bm = s1 / f(n)
    bv = (s2 - f(n) * bm * bm) / f(n - 1)
    cnt, tot = f(1e-4), f(1e-4 + n)
    delta = bm - f(0)
    return f((f(1) * cnt + bv * f(n)) + ((delta * delta) * cnt * f(n)) / tot) / tot

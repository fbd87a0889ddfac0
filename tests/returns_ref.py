"""The actor-critic return pass (`a2c_prepare`, csrc/a2c.cu) restated for the edge tests.  TEST INFRASTRUCTURE ONLY.

- A mirror of `lambda_returns_kernel`'s split: windows of 256 steps walked right to left, 32 lanes of 8 steps each.
- The per-row bar: every return is judged against its own no-cancellation scale S_t, not against the batch's largest |R|.
- The cases of tests/test_returns_edges_gpu.py and their batches: dones and reward spikes placed on the split's boundaries.
- A plain float32 recursion and mutations of it (tests/test_returns_edges.py shows the bar passes the one and fails the others).
- The DQN family's TD(λ) scan (td_lambda_kernel, the same split): its bar and scale, the cases of tests/test_td_target_edges_gpu.py and their
  batches (cuts, stale restarts, dones and spikes on the edges), ret_ms_step's choice of moment kernel, and the scan's float32 recursion and its
  mutations (tests/test_td_target_edges.py).
"""
from __future__ import annotations

import numpy as np

LAM_CHUNK, LAM_WINDOW = 8, 256      # kLamChunk, kLamWindow = 32 x kLamChunk of csrc/a2c.cu
LAM_WARPS = 8                       # kLamWarps: sequences (warps) per block
RET_STRIDE = 64 * 256               # ret_moments_kernel's grid stride (kRetBlocks x 256 threads, csrc/retms.cuh)
U32 = 2.0 ** -24                    # float32 unit roundoff
D = 5                               # observation width of the return cases


# ---- the split -----------------------------------------------------------------------------------------------------------------------------------
def windows(T):
    """(w0, len) of every window, in the kernel's order (right to left)"""
    return [(w0, min(LAM_WINDOW, T - w0)) for w0 in range(((T - 1) // LAM_WINDOW) * LAM_WINDOW, -1, -LAM_WINDOW)]


def lanes(length):
    """[lo, hi) of each of the 32 lanes in a window of `length` steps (hi <= lo: the lane has no step)"""
    return [(lane * LAM_CHUNK, min(lane * LAM_CHUNK + LAM_CHUNK, length)) for lane in range(32)]


def lane_edge(w0, length):
    """a chunk edge inside the window away from its ends: the first step of lane min(16, ·)'s chunk (None when only lane 0 has steps)"""
    k = min(16, (length - 1) // LAM_CHUNK)
    return w0 + LAM_CHUNK * k if k >= 1 else None


def edges(T):
    """the window starts that receive a carry: every w0 > 0"""
    return [w0 for w0, _ in windows(T) if w0 > 0]


# ---- the per-row bar -----------------------------------------------------------------------------------------------------------------------------
def tau(T, gamma, lam):
    """8 float32 roundings of every term along the horizon min(T, 1/(1 - γλ)), and never below 1e-5"""
    b = gamma * lam
    horizon = T if b >= 1.0 else min(T, 1.0 / (1.0 - b))
    return max(1e-5, 8 * U32 * horizon)


def lambda_scale(rew, done, v, lam, gamma):
    """S_t = |m_t r_t| + γ(1-λ)|m_{t+1} V_{t+1}| + γλ S_{t+1}, S_T = 0, float64: rew (T, ...), done and v (T+1, ...)"""
    r = np.asarray(rew, np.float64)
    T = r.shape[0]
    m = 1.0 - np.asarray(done, np.float64)
    mv = np.abs(m * np.asarray(v, np.float64))
    out = np.zeros_like(r)
    nxt = np.zeros_like(r[0])
    for t in reversed(range(T)):
        boot = mv[t + 1] if t + 1 < T else 0.0
        nxt = np.abs(m[t] * r[t]) + gamma * (1.0 - lam) * boot + gamma * lam * nxt
        out[t] = nxt
    return out


def nstep_tau(T, n):
    return max(1e-5, 8 * U32 * min(T, n + 1))


def nstep_scale(rew, done, v, n, gamma):
    """Σ_{k<n, t+k<T} γ^k |m r_{t+k}| + [t+n < T] γ^n |m V_{t+n}|, float64: the n-step return's terms without cancellation"""
    r = np.asarray(rew, np.float64)
    T = r.shape[0]
    m = 1.0 - np.asarray(done, np.float64)
    mr, mv = np.abs(m[:T] * r), np.abs(m * np.asarray(v, np.float64))[:T]
    out = np.zeros_like(r)
    for k in range(min(n, T)):
        out[: T - k] += gamma ** k * mr[k:]
    if n < T:
        out[: T - n] += gamma ** n * mv[n:]
    return out


def worst(got, want, scale, bar):
    """max over rows of |got - want| / (bar x S_t); a row with S_t = 0 (every term masked) must be exact"""
    err = np.abs(np.asarray(got, np.float64) - want)
    ratio = np.where(scale > 0, err / (bar * np.where(scale > 0, scale, 1.0)), np.where(err > 0, np.inf, 0.0))
    return float(ratio.max())


# ---- the cases -----------------------------------------------------------------------------------------------------------------------------------
# (T, N, block class of N·P mod 8, N = 32 case): every T of the sweep; N·P ≡ 1 (mod 8) leaves the last 8-warp block with one busy warp
LAMBDA_TS = (7, 8, 9, 15, 16, 17, 255, 256, 257, 511, 512, 513, 769, 1025)
LAMBDA_CASES = [(7, 1, 1), (8, 3, 0), (9, 1, 1), (15, 2, 0), (16, 3, 1), (17, 1, 0), (255, 1, 1), (256, 2, 0), (257, 3, 1), (257, 32, 0),
                (511, 1, 0), (512, 1, 1), (513, 2, 0), (769, 1, 1), (1025, 1, 0)]
GAMMAS, LAMBDAS = (0.99, 0.999), (0.0, 0.5, 0.95, 1.0)


def done_at(T):
    """the done index of each env of a λ case (None: the episode runs to T unterminated and untruncated, T: it terminates exactly at T):
    every window edge w0 - 1, w0, w0 + 1, each window's lane edge and its neighbours, and T - 1"""
    out = [None, T]
    for w0 in edges(T):
        out += [w0 - 1, w0, w0 + 1]
    for w0, length in windows(T):
        x = lane_edge(w0, length)
        if x is not None:
            out += [x - 1, x, x + 1]
    out.append(T - 1)
    seen, keep = set(), []
    for d in out:
        if (d is None or 1 <= d <= T) and d not in seen:
            seen.add(d); keep.append(d)
    return keep


def case_P(T, N, block):
    """the fewest envs >= len(done_at(T)) with N·P in the block class (1: ≡ 1 mod 8, 0: ≡ 0 mod 8)"""
    P = len(done_at(T))
    while (N * P) % 8 != block:
        P += 1
    return P


def spikes_at(T):
    """the steps that get a large reward: each window edge and its neighbours, each window's lane edge.  An off-by-one of the split at one of
    them moves a return by a whole spike, far more than the bar; away from them the rewards are small, so few spikes share a horizon."""
    out = set()
    for w0 in edges(T):
        out |= {w0 - 1, w0, w0 + 1}
    for w0, length in windows(T):
        x = lane_edge(w0, length)
        if x is not None:
            out.add(x)
    return sorted(t for t in out if 0 <= t < T)


def lambda_batch(rng, T, N, P, A=3):
    """a device-layout batch of P envs (numpy): env e's episode ends at done_at(T)[e] (the extra envs end at random steps); rewards of even (env +
    agent) are sparse and positive like LBF's and RWARE's, of odd ones dense and of either sign; every env has the spikes of spikes_at(T)"""
    obs = (rng.integers(-1, 8, size=(P, N, T + 1, D)) / 4.0).astype(np.float32)
    act = rng.integers(0, A, size=(P, N, T)).astype(np.int32)
    sparse = (rng.random((P, N, T)) < 0.2) * rng.random((P, N, T)) * 0.1
    dense = rng.standard_normal((P, N, T)) * 0.1
    parity = (np.arange(P)[:, None] + np.arange(N)[None, :]) % 2
    rew = np.where(parity[:, :, None] == 0, sparse, dense)
    sp = spikes_at(T)
    rew[:, :, sp] += rng.uniform(5.0, 10.0, size=(P, N, len(sp)))
    rew = rew.astype(np.float32)
    done = np.zeros((P, T + 1), np.uint8); filled = np.zeros((P, T), np.uint8)
    ends = done_at(T)
    for e in range(P):
        end = ends[e] if e < len(ends) else int(rng.integers(1, T + 1))
        filled[e, : T if end is None else end] = 1
        if end is not None:
            done[e, end] = 1
    return dict(obs=obs, act=act, rew=rew, done=done, filled=filled)


def sequences(s, v=None):
    """the (T, P, N) float64 rewards, (T+1, P, N) dones of a device-layout batch, and v (T+1, P, N) (given, or none)"""
    rew = s["rew"].astype(np.float64).transpose(2, 0, 1)
    done = np.repeat(s["done"].astype(np.float64).T[:, :, None], rew.shape[2], axis=2)
    return rew, done, v


def reaches(T, N, P, block):
    """the boundaries a λ case reaches, by the mirror of the split"""
    ws = windows(T)
    ends = done_at(T)
    got = {f"windows={len(ws)}", f"NP%8={(N * P) % 8}"}
    if (N * P) % 8 == block:
        got.add("block class")
    if any(length == 1 for _, length in ws):
        got.add("one-step window")
    if ws[0][1] == LAM_WINDOW:
        got.add("full last window")
    if len(ws) >= 3:
        got.add(">= 3 windows")
    for w0 in edges(T):
        for k, name in ((-1, "done at w0 - 1"), (0, "done at w0"), (1, "done at w0 + 1")):
            if w0 + k in ends:
                got.add(name)
    for w0, length in ws:
        x = lane_edge(w0, length)
        if x is not None and x in ends and (x - 1) in ends and (x + 1 in ends or x + 1 > T):
            got.add("done at a chunk edge")
    if None in ends:
        got.add("untruncated full-length episode")
    if T % LAM_CHUNK in (1, 7, 0):
        got.add({1: "one-step lane chunk", 7: "partial lane chunk", 0: "full lane chunks"}[T % LAM_CHUNK])
    if N == 32:
        got.add("N = 32")
    return got


# ---- a plain float32 recursion and its mutations -------------------------------------------------------------------------------------------------
def coefs(lam, gamma):
    """the kernel's float32(γ(1 - λ)), float32(γλ) from float32 γ and λ"""
    g, l_ = float(np.float32(gamma)), float(np.float32(lam))
    return np.float32(g * (1.0 - l_)), np.float32(g * l_)


def f32_terms(rew, done, v, lam, gamma, ignore_done_at=()):
    """a_t = m_t r_t + float32(γ(1-λ)) m_{t+1} V_{t+1} in float32, (T, ...); `ignore_done_at`: steps t whose m_{t+1} is taken as 1"""
    cv, _ = coefs(lam, gamma)
    r = np.asarray(rew, np.float32)
    T = r.shape[0]
    m = (1.0 - np.asarray(done, np.float32)).astype(np.float32)
    vv = np.asarray(v, np.float32)
    a = r * m[:T]
    boot = np.zeros_like(a)
    mb = m[1:T + 1].copy()
    for t in ignore_done_at:
        if t + 1 < T:
            mb[t] = 1.0
    boot[: T - 1] = (cv * vv[1:T]) * mb[: T - 1]
    return (a + boot).astype(np.float32)


def f32_recursion(rew, done, v, lam, gamma, next_of=None, ignore_done_at=()):
    """R_t = a_t + float32(γλ) R_{t+1} sequentially in float32.  next_of: {t: callable(R) -> the value used as R_{t+1} at step t} (mutations)"""
    _, cr = coefs(lam, gamma)
    a = f32_terms(rew, done, v, lam, gamma, ignore_done_at)
    T = a.shape[0]
    R = np.zeros((T + 1,) + a.shape[1:], np.float32)
    for t in reversed(range(T)):
        nxt = next_of[t](R) if next_of and t in next_of else R[t + 1]
        R[t] = a[t] + cr * nxt
    return R[:T]


def mutations(T, done_rows):
    """{name: f32_recursion keyword arguments} of the split's plausible defects that apply at T (done_rows: the done indices present)"""
    out = {}
    es = edges(T)
    if es:
        E = es[-1]   # the leftmost edge: the carry into window 0
        length = dict(windows(T))[E]
        lo31 = E + LAM_CHUNK * 31
        out["carry dropped at the window edge"] = dict(next_of={E - 1: lambda R: np.zeros_like(R[0])})
        out["carry from lane 31"] = dict(next_of={E - 1: (lambda R, x=(lo31 if lo31 < E + length else E + length): R[x])})
        out["window edge shifted by one"] = dict(next_of={E - 1: lambda R, x=min(E + 1, T): R[x]})
        hit = [w0 - 1 for w0 in es if w0 in done_rows]
        if hit:
            out["done[t+1] ignored on a window's last step"] = dict(ignore_done_at=hit)
    for w0, length in windows(T):
        x = lane_edge(w0, length)
        if x is not None:
            out["a lane's chunk replayed from R of the wrong step"] = dict(next_of={x - 1: lambda R, y=min(x + 1, T): R[y]})
            break
    return out


# ---- the running return statistics -------------------------------------------------------------------------------------------------------------
class StatsRef:
    """RunningMeanStd (oracle.learner_ref.RunningMeanStdRef) in float64, with the bar each update's running statistics are held to.

    The count: exact.  The mean: 1e-6 of |mean| + its spread.  The variance: 1e-6 relative, plus the eight float32 roundings of the update
    itself (8u relative), plus what the float32 update of the reference (and of ret_ms_update_kernel, which keeps its operation order) loses in
    delta = batch_mean - mean.  Both are float32 (the running mean carries its own rounding from earlier updates), so delta is off by up to
    2u(|batch_mean| + |mean|), which moves var by 2 |delta| times that, times count n / (count + n)².  The running statistics carry the earlier
    updates' bars, weighted count / (count + n).  Returns with a large mean and a batch mean that moves between updates make those terms the
    larger ones.

    `err`: a per-return bound on the returns themselves (the λ-returns' τ S_t, where rounding accumulates along a sequence): the batch mean
    moves by up to its mean, the batch variance by up to 2 spread rms(err) + mean(err²) (Cauchy-Schwarz).  Without it the returns are taken
    as exact: one or two roundings per return, uncorrelated with the returns, average out of the moments."""

    def __init__(self, n):
        import torch

        from oracle import learner_ref as lr

        self._torch = torch
        self.rms = lr.RunningMeanStdRef((n,))
        self.rms.mean, self.rms.var = self.rms.mean.double(), self.rms.var.double()
        self.var_bar = self.mean_bar = None

    def update(self, x, err=None):
        """absorb the float64 returns x (rows, n), each known to within err (rows, n) or exactly"""
        x = np.asarray(x, np.float64).reshape(-1, np.shape(x)[-1])
        mean0, cnt, n = self.rms.mean.numpy().copy(), self.rms.count, x.shape[0]
        bm, bv = x.mean(0), x.var(0, ddof=1) if n > 1 else np.zeros(x.shape[1])
        e = np.zeros_like(x) if err is None else np.asarray(err, np.float64).reshape(x.shape)
        e_mean, e_var = e.mean(0), 2 * np.sqrt(bv * (e ** 2).mean(0)) + (e ** 2).mean(0)
        tot = cnt + n
        old_m, old_v = (0.0, 0.0) if self.mean_bar is None else (self.mean_bar, self.var_bar)
        self.rms.update(self._torch.tensor(x))
        var = self.rms.var.numpy()
        self.mean_bar = 1e-6 * (np.abs(self.rms.mean.numpy()) + np.sqrt(var)) + old_m * cnt / tot + e_mean * n / tot
        self.var_bar = ((1e-6 + 8 * U32) * var + old_v * cnt / tot + e_var * n / tot
                        + 2 * np.abs(bm - mean0) * (2 * U32 * (np.abs(bm) + np.abs(mean0)) + e_mean) * cnt * n / tot ** 2)

    @property
    def mean(self):
        return self.rms.mean.numpy()

    @property
    def var(self):
        return self.rms.var.numpy()

    @property
    def count(self):
        return self.rms.count


# ---- the DQN family's TD(λ) targets (td_lambda_kernel, col_td_kernel and ret_ms_step, csrc/dqn.cu) --------------------------------------------------
# td_lambda_kernel splits each (column, episode) sequence as lambda_returns_kernel does: windows of LAM_WINDOW steps right to left, lanes of
# LAM_CHUNK; it runs TDL_WARPS sequences per block.  col_td_kernel, which writes the bootstrap values and the TD error, and its block_loss_part run
# one thread per (c, b, t) in blocks of COL_BLOCK.
TDL_WARPS = 8                       # kTdlWarps
COL_BLOCK = 256                     # col_td_kernel's block
RET_COLS_N, RET_COLS_PT = 64, 1024  # ret_ms_step takes ret_moments_cols_kernel when N > 64 and P·T <= 1024


def td_tau(T, gamma, lam):
    """the TD(λ) target's bar: 16 float32 roundings of every term along the horizon min(T, 1/(1 - γλ)), never below 2e-5 -- twice tau's.  The
    rounding of float32(γλ) compounds along the chain (about horizon / 2 roundings on the farthest terms, which a plain float32 recursion shows
    at 20 u for a horizon of 17), and each step rounds b_t = r_t + (γ (1 - d_{t+1})) ((1 - λ f_{t+1}) v_{t+1}) four times."""
    return 2 * tau(T, gamma, lam)


def td_columns(kind, N):
    """C of a DQN-family learner: IDQN one column per agent, VDN and QMIX one column of the team"""
    return N if kind == "idqn" else 1


def ret_ms_path(kind, N, B, T):
    """the moment kernel ret_ms_step launches for a standardised update: VDN and QMIX keep one statistic per batch entry (N = B columns of P = 1
    episode of T returns), IDQN one per agent (N columns of P = B episodes)"""
    n, P = (B, 1) if kind != "idqn" else (N, B)
    return "cols" if n > RET_COLS_N and P * T <= RET_COLS_PT else "grid"


def td_lambda_scale(rew, done, filled, boot, lam, gamma):
    """S_t = |r_t| + γ (1 - d_{t+1}) (|1 - λ f_{t+1}| |v_{t+1}| + λ f_{t+1} S_{t+1}), f_T = 0, float64: the TD(λ) target's terms without
    cancellation, cut at the first unfilled row as the target is.  rew, filled, boot (T, ...) with boot[t] = v_{t+1}; done (T+1, ...)"""
    r, v = np.abs(np.asarray(rew, np.float64)), np.abs(np.asarray(boot, np.float64))
    d, f = np.asarray(done, np.float64), np.asarray(filled, np.float64)
    T = r.shape[0]
    out, nxt = np.zeros_like(r), np.zeros_like(r[0])
    for t in reversed(range(T)):
        f1 = f[t + 1] if t + 1 < T else 0.0
        nxt = r[t] + gamma * (1.0 - d[t + 1]) * (np.abs(1.0 - lam * f1) * v[t] + lam * f1 * nxt)
        out[t] = nxt
    return out


def td_rows(T):
    """the rows that get an event: every window edge w0 - 1, w0, w0 + 1, each window's lane edge and its neighbours, and T - 1 (inside [1, T))"""
    out = []
    for w0 in edges(T):
        out += [w0 - 1, w0, w0 + 1]
    for w0, length in windows(T):
        x = lane_edge(w0, length)
        if x is not None:
            out += [x - 1, x, x + 1]
    out.append(T - 1)
    return sorted({x for x in out if 1 <= x < T})


TD_EVENTS = ("cut", "done", "stale")


def td_episodes(T):
    """the scripted episodes of a TD(λ) case, (kind, row): one filled to T without a done flag, one terminated at T, and per row x of td_rows(T)
    - cut: filled up to x (x is the first unfilled row), no done flag: a truncated episode;
    - done: terminated at x (done[x] = 1), unfilled from x;
    - stale: filled up to x - 2, row x - 1 unfilled, filled again from x (a re-used slot's stale tail restarts at x), random done flags in it."""
    return [("full", T), ("done", T)] + [(k, x) for x in td_rows(T) for k in TD_EVENTS]


def td_batch(rng, T, N, B, A=6, D=D):
    """a device-layout store of B episodes: the first len(td_episodes(T)) are scripted, the rest end at random steps; rewards as lambda_batch's
    (sparse and dense, spikes on the window and lane edges); VDN and QMIX read agent 0's reward"""
    obs = (rng.integers(-1, 8, size=(B, N, T + 1, D)) / 4.0).astype(np.float32)
    act = rng.integers(0, A, size=(B, N, T)).astype(np.int32)
    sparse = (rng.random((B, N, T)) < 0.2) * rng.random((B, N, T)) * 0.1
    dense = rng.standard_normal((B, N, T)) * 0.1
    parity = (np.arange(B)[:, None] + np.arange(N)[None, :]) % 2
    rew = np.where(parity[:, :, None] == 0, sparse, dense)
    sp = spikes_at(T)
    rew[:, :, sp] += rng.uniform(5.0, 10.0, size=(B, N, len(sp)))
    done = np.zeros((B, T + 1), np.uint8); filled = np.zeros((B, T), np.uint8)
    eps = td_episodes(T)
    for e in range(B):
        kind, x = eps[e] if e < len(eps) else (("done", "cut")[e % 2], int(rng.integers(1, T + 1)))
        if kind == "stale":
            filled[e, : max(x - 1, 0)] = 1
            filled[e, x:] = 1
            done[e, x + 1:] = rng.random(T - x) < 0.2
        else:
            filled[e, :x] = 1
            done[e, x] = kind == "done"
    return dict(obs=obs, act=act, rew=rew.astype(np.float32), done=done, filled=filled)


def td_sequences(s, C):
    """(rew, done, filled) of a device-layout store in time-major float64, (T, C, B) and done (T+1, C, B): column c reads agent c's reward (C = 1:
    agent 0's), every column of an episode its done and filled flags"""
    rew = s["rew"][:, :C].astype(np.float64).transpose(2, 1, 0)
    B, T = s["filled"].shape
    done = np.broadcast_to(s["done"].astype(np.float64).T[:, None, :], (T + 1, C, B))
    filled = np.broadcast_to(s["filled"].astype(np.float64).T[:, None, :], (T, C, B))
    return rew, done, filled


def td_case_B(T, C, cb8, cbt=None):
    """the fewest episodes >= len(td_episodes(T)) with C·B ≡ cb8 (mod 8) and, when given, C·B·T ≡ cbt (mod COL_BLOCK)"""
    B = len(td_episodes(T))
    while (C * B) % 8 != cb8 or (cbt is not None and (C * B * T) % COL_BLOCK != cbt):
        B += 1
    return B


# (T, kind, N, C·B mod 8 or None for C·B < 8, C·B·T mod 256 or None): every T mod 256 in {1, 7, 8, 9, 255, 0}, 1 to 5 windows
TD_CASES = [(1, "idqn", 2, None, None), (7, "vdn", 2, 1, 255), (9, "qmix", 2, 7, None), (255, "idqn", 3, 0, None), (256, "qmix", 2, 1, 0),
            (257, "vdn", 2, 7, 255), (263, "idqn", 3, 1, None), (264, "qmix", 3, 0, None), (265, "vdn", 2, 1, 1), (511, "qmix", 2, 7, None),
            (512, "idqn", 3, 7, None), (769, "vdn", 2, 0, None), (1024, "qmix", 2, 1, None), (1025, "idqn", 3, 1, None)]


def td_case(T, kind, N, cb8, cbt):
    """(C, B) of a TD(λ) case; C·B < 8: three episodes of one row (T = 1 has no edge rows)"""
    C = td_columns(kind, N)
    return C, (3 if cb8 is None else td_case_B(T, C, cb8, cbt))


def td_reaches(T, kind, N, B, standardise=False):
    """the boundaries a TD(λ) case reaches, by the mirror of the split"""
    C = td_columns(kind, N)
    ws = windows(T)
    got = {f"windows={len(ws)}", f"CB%8={(C * B) % 8}", f"T%256={T % LAM_WINDOW}"}
    if C * B < 8:
        got.add("CB<8")
    if (C * B) % TDL_WARPS and C * B > TDL_WARPS:
        got.add("partial last block")
    if (C * B * T) % COL_BLOCK in (COL_BLOCK - 1, 0, 1):
        got.add(f"CBT%256={(C * B * T) % COL_BLOCK}")
    eps = td_episodes(T)[:B]
    first_unfilled = {x for k, x in eps if k in ("cut", "done") and x < T} | {x - 1 for k, x in eps if k == "stale"}
    restarts = {x for k, x in eps if k == "stale"}
    dones = {x for k, x in eps if k == "done"}
    for w0 in edges(T):
        for name, rows in (("cut", first_unfilled), ("restart", restarts), ("done", dones)):
            got |= {f"{name} at w0{k:+d}" if k else f"{name} at w0" for k in (-1, 0, 1) if w0 + k in rows}
    for w0, length in ws:
        x = lane_edge(w0, length)
        if x is not None:
            for name, rows in (("cut", first_unfilled), ("restart", restarts), ("done", dones)):
                if x in rows:
                    got.add(f"{name} at a lane edge")
    if standardise:
        got.add(f"ret_ms {ret_ms_path(kind, N, B, T)}")
    return got


def td_f32_recursion(rew, done, filled, boot, lam, gamma, next_of=None, f_from_t=False, ignore_cut_at=()):
    """td_lambda_kernel's arithmetic done sequentially in float32: a_t = float32(γλ) (1 - d_{t+1}) f_{t+1}, b_t = r_t + (γ (1 - d_{t+1})) ((1 - λ
    f_{t+1}) v_{t+1}), G_t = b_t + a_t G_{t+1}.  Mutations: next_of {t: callable(G) -> the value used as G_{t+1}}; f_from_t: f_{t+1} read as f_t;
    ignore_cut_at: steps t whose f_{t+1} is taken as 1"""
    g, l_ = np.float32(gamma), np.float32(lam)
    gl = np.float32(float(g) * float(l_))
    r, v = np.asarray(rew, np.float32), np.asarray(boot, np.float32)
    d, f = np.asarray(done, np.float32), np.asarray(filled, np.float32)
    T = r.shape[0]
    G = np.zeros((T + 1,) + r.shape[1:], np.float32)
    one = np.float32(1.0)
    for t in reversed(range(T)):
        live = one - d[t + 1]
        f1 = (f[t] if f_from_t else f[t + 1]) if t + 1 < T else np.zeros_like(r[0])
        if t in ignore_cut_at:
            f1 = np.ones_like(f1)
        a = gl * live * f1
        b = r[t] + (g * live) * ((one - l_ * f1) * v[t])
        nxt = next_of[t](G) if next_of and t in next_of else G[t + 1]
        G[t] = b + a * nxt
    return G[:T]


def td_mutations(T, cut_rows):
    """{name: td_f32_recursion keyword arguments} of td_lambda_kernel's plausible defects that apply at T (cut_rows: the first unfilled rows present)"""
    out = {"f_{t+1} read as f_t": dict(f_from_t=True)} if cut_rows else {}
    es = edges(T)
    if es:
        E = es[-1]
        out["carry between windows dropped"] = dict(next_of={w0 - 1: lambda G: np.zeros_like(G[0]) for w0 in es})
        out["window edge shifted by one"] = dict(next_of={E - 1: lambda G, x=min(E + 1, T): G[x]})
        hit = [w0 - 1 for w0 in es if w0 in cut_rows]
        if hit:
            out["cut ignored on a window's last step"] = dict(ignore_cut_at=hit)
    wrong = {}
    for w0, length in windows(T):   # every lane but the last two takes G after the lane two to its right; lanes 30 and 31 the carry
        for lane in range(32):
            lo, hi = lane * LAM_CHUNK, min(lane * LAM_CHUNK + LAM_CHUNK, length)
            if lo < hi and hi < length:
                wrong[w0 + hi - 1] = lambda G, x=w0 + min((lane + 2) * LAM_CHUNK, length) if lane < 30 else w0 + length: G[x]
    if wrong:
        out["a lane's incoming G from two lanes over"] = dict(next_of=wrong)
    return out

"""The update tail every learner ends in, in float64 -- the reduction of the per-CTA gradient partials, the loss statistics, clip_grad_norm_, the
optimiser step and the target update -- and the cases that reach every edge of its split on a device of capacity C.  TEST INFRASTRUCTURE ONLY.

The tail runs as one of three paths (marl_debug_tail_run):
  0  reduce_adam_kernel<0>: pb parameters x ns CTA-slices per block, one co-resident wave, a grid barrier between the sums and the step;
  1  grad_reduce_kernel (64 parameters x 16 slices per block) + adam_kernel with the per-block sums of squares (the DQN family's fallback);
  2  the same without them: adam_kernel's float4 norm (actor-critic learners, marl_dqn_update_apply, the QMIX mixer's step).
tail_shape restates reduce_adam_shape; reduce_ref and step_ref are the tail in float64; cases(n_sm, capacity) lists what
tests/test_optimizer_tail_gpu.py runs, each case with the edges it claims, and reaches() says which edges a case reaches."""
from __future__ import annotations

import dataclasses
import math

import numpy as np

U = 2.0 ** -24   # float32 unit round-off
OPTS = ("Adam", "AdamW", "RMSprop", "Adagrad", "SGD")   # MARL_OPT_* order
DEFAULTS = {"Adam": dict(beta1=0.9, beta2=0.999, eps=1e-8), "AdamW": dict(beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=1e-2),
            "RMSprop": dict(alpha=0.99, eps=1e-8), "Adagrad": dict(eps=1e-10), "SGD": dict()}
USES_M = {"Adam", "AdamW"}
USES_V = {"Adam", "AdamW", "RMSprop", "Adagrad"}
MIN_PB, MAX_PB, MAX_NS, THREADS = 128, 512, 4, 1024
REDUCE_SLICES, FUSED_ROUND = 16, 20   # grad_reduce_kernel's slices; reduce_adam_kernel's loads per slice per round


def f32(x):
    return float(np.float32(x))


# ---- the block shape -------------------------------------------------------------------------------------------------------------------------------
def tail_shape(n, capacity):
    """reduce_adam_shape: (pb, ns), or None when the learners take the two-kernel tail"""
    pb = (-(-n // capacity) + 31) // 32 * 32
    if pb < MIN_PB or pb > MAX_PB:
        return None
    ns = min(THREADS // pb, MAX_NS)
    return (pb, ns) if ns >= 2 else None


# ---- float64 reference -----------------------------------------------------------------------------------------------------------------------------
def reduce_ref(scratch, ctas, P, loss_part, n_loss_parts, stats_in, accumulate):
    """(gradient sums [n_nets * P], the 4 statistics): network k's partials are scratch rows [cta_begin[k], cta_begin[k+1])"""
    begin = np.concatenate([[0], np.cumsum(ctas)])
    g = np.concatenate([scratch[begin[k]:begin[k + 1], :P].astype(np.float64).sum(0) for k in range(len(ctas))])
    st = loss_part[:n_loss_parts].astype(np.float64).sum(0)
    if accumulate:
        st = st + np.asarray(stats_in, np.float64)
    return g, st


def step_consts(opt, lr, step):
    """set_step_consts: the float32 constants of one step (betas as float32; bias corrections, AdamW's decay and RMSprop's 1 - alpha in double,
    rounded once)"""
    d = DEFAULTS[opt]
    c = dict(lr=f32(lr), eps=f32(d.get("eps", 0.0)), bc1=1.0, bc2_sqrt=1.0, decay=1.0, beta1=0.0, beta2=0.0)
    if opt in ("Adam", "AdamW"):
        b1, b2 = f32(d["beta1"]), f32(d["beta2"])
        c.update(beta1=b1, beta2=b2, bc1=f32(1.0 - b1 ** step), bc2_sqrt=f32(math.sqrt(1.0 - b2 ** step)))
        if opt == "AdamW":
            c["decay"] = f32(1.0 - f32(lr) * d["weight_decay"])
    elif opt == "RMSprop":
        c.update(beta2=f32(d["alpha"]), beta1=f32(1.0 - d["alpha"]))
    return c


def clip_coef(norm, grad_clip):
    """torch.nn.utils.clip_grad_norm_'s coefficient"""
    return min(grad_clip / (norm + 1e-6), 1.0) if grad_clip > 0 else 1.0


def device_clip(norm32, grad_clip):
    """the coefficient the kernels derive from their float32 norm: fminf(grad_clip / (norm + 1e-6f), 1) in float32"""
    if not grad_clip > 0:
        return np.float32(1.0)
    return min(np.float32(grad_clip) / (np.float32(norm32) + np.float32(1e-6)), np.float32(1.0))


def opt_step(opt, c, g, m, v, th):
    """one step in float64 with the constants c of step_consts -> (theta, m, v, no-cancellation scale of the update)"""
    g, m, v, th = (np.asarray(x, np.float64) for x in (g, m, v, th))
    if opt in ("Adam", "AdamW"):
        th = th * c["decay"]
        m2 = m + (g - m) * (1.0 - c["beta1"])
        v2 = v * c["beta2"] + g * g * (1.0 - c["beta2"])
        denom = np.sqrt(v2) / c["bc2_sqrt"] + c["eps"]
        upd = (c["lr"] / c["bc1"]) * (m2 / denom)
        scale = (c["lr"] / c["bc1"]) * (np.abs(m) + np.abs(g - m) * (1.0 - c["beta1"])) / denom
        return th - upd, m2, v2, scale
    if opt in ("RMSprop", "Adagrad"):
        v2 = c["beta1"] * g * g + v * c["beta2"] if opt == "RMSprop" else g * g + v
        upd = c["lr"] * g / (np.sqrt(v2) + c["eps"])
        return th - upd, m, v2, np.abs(upd)
    upd = c["lr"] * g
    return th - upd, m, v, np.abs(upd)


def step_ref(grad, stats, theta, m, v, tgt, opt, lr, grad_clip, step, target, tau, clip=None):
    """The step after the reduction, in float64, from the reduced gradient `grad` [n] and `stats` [4].  clip = None: the exact coefficient of
    clip_grad_norm_ and g = grad / fill * clip; clip = a float32 coefficient: g exactly as the kernels form it, (grad * (1 / fill)) * clip in
    float32 (then every error left is the step's own).  target = (mode, begin, count).  Returns the new state, norm, clip, loss_out and the
    update's scale."""
    fill = float(stats[1])
    grad = np.asarray(grad, np.float64)
    norm = math.sqrt(float((grad * grad).sum())) / fill
    if clip is None:
        coef = clip_coef(norm, grad_clip)
        g = grad / fill * coef
    else:
        coef = float(clip)
        g = ((np.asarray(grad, np.float32) * (np.float32(1.0) / np.float32(fill))) * np.float32(clip)).astype(np.float64)
    c = step_consts(opt, lr, step)
    th, m2, v2, scale = opt_step(opt, c, g, m, v, theta)
    mode, begin, count = target
    tgt2 = np.asarray(tgt, np.float64).copy()
    if mode == 1:
        tgt2[:count] = th[begin:begin + count]
    elif mode == 2:
        tgt2[:count] = (1.0 - f32(tau)) * tgt2[:count] + f32(tau) * th[begin:begin + count]
    loss_out = np.array([stats[0] / fill, norm, stats[2] / fill, stats[3] / fill, fill, 0.0])
    return dict(theta=th, m=m2, v=v2, tgt=tgt2, norm=norm, clip=coef, g=g, loss_out=loss_out, scale=scale, consts=c, m_old=np.asarray(m, np.float64),
                v_old=np.asarray(v, np.float64))


# ---- bars ------------------------------------------------------------------------------------------------------------------------------------------
def norm_chain(path, n, ns_shape=None):
    """The longest chain of float32 additions a square passes through on its way into the norm, by path (the norm's relative bar is this + 8 units:
    the square, sqrt, the division by fill and the slack of a first-order bound).
    0: a 32-lane shuffle tree (5), the block's pb / 32 warp partials in order, lane k's blocks k, k + 32, ..., a shuffle tree (5);
    1: grad_reduce_kernel's sq[t] + sq[t + 32] and shuffle tree (6), then adam_kernel's thread-serial walk over the block sums and its 8-level tree;
    2: adam_kernel's thread-serial walk over ceil(n / 1024) float4 groups (4 each) plus the scalar tail, and the 8-level tree."""
    if path == 0:
        pb, _ = ns_shape
        grid = -(-n // pb)
        return 5 + pb // 32 + -(-grid // 32) + 5
    if path == 1:
        return 6 + -(-(-(-n // 64)) // 256) + 8
    return 4 * -(-(n // 4) // 256) + 1 + 8


def norm_bar(path, n, shape=None):
    return (norm_chain(path, n, shape) + 8) * U


def step_bars(opt, ref, theta, tgt_old, tau, target):
    """element-wise bars of the step given the kernels' own g (step_ref with clip = the device coefficient): a few units of each term's no-
    cancellation scale.  m, v: 12 units of the terms of one update (up to 4 roundings, three times over for slack); theta: its own rounding and AdamW's decay
    (4 units of |theta| before and after) and 16 units of the update's scale (m and v carry 4, sqrt, the two divisions and eps 1 each); a Polyak target: 8 units
    of its two terms (1 - tau, two products and the sum round) plus tau x theta's bar."""
    th0 = np.abs(np.asarray(theta, np.float64))
    g = np.abs(ref["g"])
    c = ref["consts"]
    out = {"theta": 4 * U * (th0 + np.abs(ref["theta"])) + 16 * U * ref["scale"]}
    if opt in USES_M:
        out["m"] = 12 * U * (np.abs(ref["m_old"]) + g * (1 - c["beta1"]) + np.abs(ref["m"]))
    if opt in USES_V:
        out["v"] = 12 * U * (np.abs(ref["v"]) + np.abs(ref["v_old"]))
    mode, begin, count = target
    if mode == 2:
        t = f32(tau)
        out["tgt"] = 8 * U * ((1 - t) * np.abs(tgt_old[:count]) + t * np.abs(ref["theta"][begin:begin + count])) + t * out["theta"][begin:begin + count]
    return out


def worst(got, want, bar):
    """largest |got - want| / bar (0 when all are equal)"""
    d = np.abs(np.asarray(got, np.float64) - np.asarray(want, np.float64))
    if not d.any():
        return 0.0
    return float((d / np.maximum(bar, 1e-300)).max())


# ---- the cases -------------------------------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass(frozen=True)
class Case:
    name: str
    P: int
    ctas: tuple                 # CTAs of each network (their sum: no more than the device's SMs, as the learners use)
    pitch: int                  # scratch floats per CTA (>= P; the padding [P, pitch) holds NaN)
    n_loss_parts: int
    accumulate: int
    opts: tuple
    clip: str                   # "off" (grad_clip 0, a huge norm), "below" / "above" (norm x (1 -+ 2^-10): just clipping / not), "active" (100x), "mild"
    step: int                   # 1: m = v = 0; 7: from a non-zero state
    target: tuple               # (mode, begin, count)
    paths: tuple
    claims: frozenset = frozenset()

    @property
    def n_nets(self):
        return len(self.ctas)

    @property
    def n(self):
        return self.P * len(self.ctas)


def cta_begin(ctas):
    return [0] + list(np.cumsum(ctas))


def _divisor(n, prefer):
    """the first d of `prefer` (network counts) that divides n"""
    for d in prefer:
        if d <= 32 and n % d == 0:
            return d
    return 1


_COUNTS = (1, 2, 3, 15, 16, 17, 39, 40, 41, 47, 48, 49, 59, 60, 61, 63, 64, 65, 79, 80, 81)


def _spread(n_nets, start, budget):
    """per-network CTA counts cycling through _COUNTS from `start`, within `budget` CTAs in all (every network keeps at least one)"""
    out, left = [], budget
    for k in range(n_nets):
        c = _COUNTS[(start + k) % len(_COUNTS)]
        c = max(1, min(c, left - (n_nets - k - 1)))
        out.append(c)
        left -= c
    return tuple(out)


def _target(i, n):
    """modes 0 / 1 / 2 in turn, over the slices [0, n), [0, n - n // 3) (ends before n) and [a, n) with an odd a"""
    mode = i % 3
    kind = (i // 3) % 3
    if n == 1 or kind == 0:
        return (mode, 0, n)
    if kind == 1:
        return (mode, 0, n - max(1, n // 3))
    a = (n // 4) | 1
    a = min(a, n - 1)
    return (mode, a, n - a)


def cases(n_sm, capacity):
    """every case of tests/test_optimizer_tail_gpu.py on a device of n_sm SMs and fused capacity `capacity` (= n_sm at one block per SM)"""
    C = capacity
    out = []
    parts = (1, 31, 32, 33, C)
    clips = ("off", "below", "above", "active", "mild")
    k = [0]

    def add(name, P, ctas, paths, claims=(), **kw):
        i = k[0]
        k[0] += 1
        d = dict(pitch=P + (i % 4) + (1 if P % 4 == 0 else 0), n_loss_parts=parts[i % 5], accumulate=(i // 5) % 2, clip=clips[i % 5 if i % 7 else 4],
                 step=(1, 7)[(i // 2) % 2], target=_target(i, P * len(ctas)), opts=OPTS if i % 6 == 0 else ("Adam", OPTS[1 + i % 4]))
        d.update(kw)
        out.append(Case(name, P, tuple(ctas), paths=paths, claims=frozenset(claims), **d))

    # every pb class at its low edge, one below the top and at the top (the last block full)
    for pb in range(MIN_PB, MAX_PB + 1, 32):
        for where, n in (("low", C * (pb - 32) + 1), ("top-1", C * pb - 1), ("top", C * pb)):
            nets = _divisor(n, (3, 5, 7, 2, 11, 13, 6, 4, 1) if where != "low" else (1, 2, 3))
            ctas = _spread(nets, pb // 32 + len(where), n_sm)
            add(f"pb{pb}_{where}", n // nets, ctas, (0, 1, 2), {f"pb={pb}", f"pb {where}"})
    # the two refusals: the fused kernel must not launch
    for what, n in (("pb<128", C * 96), ("pb>512", C * 512 + 1)):
        nets = _divisor(n, (2, 3, 1))
        add(f"refuse_{what}", n // nets, _spread(nets, 5, n_sm), (0, 1, 2), {f"refuse {what}"})
    # small n on the two-kernel paths: float4 groups and the scalar tail, one partial block of 64
    for n in (1, 2, 3, 4, 5, 63, 64, 65, 255, 256, 257):
        add(f"small_n{n}", n, (min(3 + n % 5, n_sm),), (1, 2), {f"n%4={n % 4}"})
    # the largest learner: 32 networks of obs 31, hidden 128, 8 actions
    P32 = 31 * 128 + 128 + 128 * 128 + 128 + 128 * 8 + 8
    add("largest_32x_obs31_h128_a8", P32, _spread(32, 0, n_sm), (1, 2), {"largest"})
    # per-network CTA counts at the edges of both reductions; several networks per block, P not a multiple of 4, 32 or pb
    for name, P, ctas, claims in (("one_net_C_ctas", 301, (n_sm,), {"C CTAs", "slice 15 used"}),
                                  ("nets_1_80", 997, (1, 80), {"a network with one CTA", "uneven split"}),
                                  ("nets_16_17_15_48", 203, (16, 17, 15, 48), {"reduce 16-1", "reduce 16+0", "reduce 16+1", "reduce 48+0"}),
                                  ("nets_39_41_47_3", 61, (39, 41, 47, 3), {"t2 leftover", "reduce 48-1", "P<64"}),
                                  ("nets_49_59_2", 257, (49, 59, 2), {"reduce 48+1", "t2 leftover"}),
                                  ("nets_60_61_1", 129, (60, 61, 1), {"a network with one CTA", "t2 leftover"}),
                                  ("nets_63_64_5_p18", 18, (63, 64, 5), {"reduce 64-1", "reduce 64+0", "P<64"}),
                                  ("nets_65_40_1", 1503, (65, 40, 1), {"reduce 64+1", "a network with one CTA"}),
                                  ("nets_79_3_3", 47, (79, 3, 3), {"P<64", "uneven split"}),
                                  ("nets_81_2_1", 4097, (81, 2, 1), {"a network with one CTA", "uneven split"})):
        if sum(ctas) <= n_sm:
            add(name, P, ctas, (0, 1, 2) if tail_shape(P * len(ctas), C) else (1, 2), claims)
    return out


# ---- which edges a case reaches --------------------------------------------------------------------------------------------------------------------
def reaches(case, capacity):
    """the edges of the split `case` reaches on a device of fused capacity `capacity`"""
    r = set()
    n, P = case.n, case.P
    shape = tail_shape(n, capacity)
    if shape is None:
        pb_raw = (-(-n // capacity) + 31) // 32 * 32
        r.add("refuse pb<128" if pb_raw < MIN_PB else "refuse pb>512")
    else:
        pb, ns = shape
        r.add(f"pb={pb}")
        r.add(f"ns={ns}")
        lo = capacity * (pb - 32) + 1
        if n == lo:
            r.add("pb low")
        if n == capacity * pb - 1:
            r.add("pb top-1")
        if n == capacity * pb:
            r.add("pb top")
        if n % pb:
            r.add("partial last block")
        if case.n_nets > 1 and any((b * pb) // P != (min((b + 1) * pb, n) - 1) // P for b in range(-(-n // pb))):
            r.add("block straddles nets")
        for c in case.ctas:
            if c < ns:
                r.add("fewer CTAs than slices")
            for e in (FUSED_ROUND * ns, 2 * FUSED_ROUND * ns):
                for dlt in (-1, 0, 1):
                    if c == e + dlt:
                        r.add(f"fused {'20' if e == FUSED_ROUND * ns else '40'}ns{dlt:+d}")
    for c in case.ctas:
        for e in (16, 48, 64):
            for dlt in (-1, 0, 1):
                if c == e + dlt:
                    r.add(f"reduce {e}{dlt:+d}")
        rem = c % (4 * REDUCE_SLICES)
        if rem > 2 * REDUCE_SLICES:   # some slice has three leftover loads (t2)
            r.add("t2 leftover")
        if c > 15:
            r.add("slice 15 used")
    if case.n_nets > 1 and len(set(case.ctas)) > 1:
        r.add("uneven split")
    if 1 in case.ctas and case.n_nets > 1:
        r.add("a network with one CTA")
    if P < 64 and case.n_nets > 1:
        r.add("P<64")
    if P % 4 and P % 32 and (shape is None or P % shape[0]):
        r.add("P odd shape")
    r.add(f"n%4={n % 4}")
    r.add(f"loss parts {case.n_loss_parts if case.n_loss_parts != capacity else 'C'}")
    r.add(f"accumulate {case.accumulate}")
    r.add(f"clip {case.clip}")
    r.add(f"step {case.step}")
    mode, begin, count = case.target
    r.add(f"target mode {mode}")
    if begin == 0 and count < n:
        r.add("target ends before n")
    if begin % 2 and begin + count == n:
        r.add("target odd start to n")
    if n == 32 * (31 * 128 + 128 + 128 * 128 + 128 + 128 * 8 + 8):
        r.add("largest")
    for c in case.ctas:
        if c == capacity:
            r.add("C CTAs")
    return r


def needed(capacity):
    """the edges the cases must reach together"""
    s = {f"pb={pb}" for pb in range(MIN_PB, MAX_PB + 1, 32)} | {"ns=2", "ns=3", "ns=4"}
    s |= {"pb low", "pb top-1", "pb top", "partial last block", "block straddles nets", "fewer CTAs than slices", "refuse pb<128", "refuse pb>512"}
    s |= {f"fused {w}ns{d:+d}" for w in ("20",) for d in (-1, 0, 1)} | {"fused 40ns+0", "fused 40ns+1"}
    s |= {f"reduce {e}{d:+d}" for e in (16, 48, 64) for d in (-1, 0, 1)} | {"t2 leftover", "slice 15 used"}
    s |= {"uneven split", "a network with one CTA", "P<64", "P odd shape", "largest", "C CTAs"}
    s |= {f"n%4={k}" for k in range(4)} | {f"loss parts {p}" for p in (1, 31, 32, 33, "C")} | {"accumulate 0", "accumulate 1"}
    s |= {f"clip {c}" for c in ("off", "below", "above", "active")} | {"step 1", "step 7"}
    s |= {"target mode 0", "target mode 1", "target mode 2", "target ends before n", "target odd start to n"}
    return s


# ---- learner configurations at each fused class ----------------------------------------------------------------------------------------------------
def dqn_params(N, D, H, A):
    """IDQN's trainable floats: N independent networks of obs D, hidden H ([H, H]) and A actions"""
    return N * (H * D + H + H * H + H + A * H + A)


def learner_cases(capacity, max_nets=4):
    """IDQN configurations (N, D, H, A) that put a real handle's tail at every fused class this capacity reaches, and around both refusals:
    {label: (N, D, H, A, n)}.  Labels: "pb=<pb>" (H = 128 where the class has one, for the tensor-core images, else the widest H), "pb=128 small
    edge" (the smallest n above C * 96), "refused below" (the largest n up to C * 96), "pb=512 top" (the largest n up to C * 512), "refused above"
    (the smallest n above C * 512).  N <= max_nets keeps the oracle small; D <= 31 (the DQN family's widest observation), 2 <= A <= 8."""
    N, D, H, A = np.meshgrid(np.arange(1, max_nets + 1), np.arange(1, 32), np.arange(1, 129), np.arange(2, 9), indexing="ij")
    N, D, H, A = (x.ravel() for x in (N, D, H, A))
    n = dqn_params(N, D, H, A)
    order = np.lexsort((A, D, N, -H))   # widest H first, then fewest networks, narrowest observation, fewest actions

    def pick(mask, key=None):
        idx = order[mask[order]]
        if not len(idx):
            return None
        if key is not None:
            idx = idx[np.argsort(key[idx], kind="stable")[:1]]
        k = idx[0]
        return (int(N[k]), int(D[k]), int(H[k]), int(A[k]), int(n[k]))

    C = capacity
    out = {}
    for pb in range(MIN_PB, MAX_PB + 1, 32):
        c = pick((n > C * (pb - 32)) & (n <= C * pb))
        if c is not None:
            out[f"pb={pb}"] = c
    out["pb=128 small edge"] = pick(n > C * 96, n)
    out["refused below"] = pick(n <= C * 96, -n)
    out["pb=512 top"] = pick(n <= C * 512, -n)
    out["refused above"] = pick(n > C * 512, n)
    return out


def ac_params(N, D, H, A):
    """IA2C's (n_actor, n_critic): N independent actors (A outputs) and critics (1 output) of obs D and hidden H"""
    return dqn_params(N, D, H, A), dqn_params(N, D, H, 1)

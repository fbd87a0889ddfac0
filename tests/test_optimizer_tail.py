"""The update tail on the CPU: what tests/test_optimizer_tail_gpu.py relies on.

- tail_ref's optimiser steps and clip coefficient are torch.optim's and clip_grad_norm_'s (float64, over a few steps of each optimiser).
- Every case the GPU test generates reaches the edges it claims on 114 SMs (H100 PCIe) and 132 SMs (H100 SXM), and together the cases reach every
  edge of the split: each pb class and both ns switches, the two refusals, the edges of both reductions' CTA loops, the scalar tail of the float4
  norm, the loss-statistics warps, the clip, the optimiser state and the target slices.
- A float32 restatement of the tail in the kernels' order of operations passes the GPU test's bars with at least 2x margin (each
  check's fraction printed with -s; the worst are the gradient sums of a network of 3 CTAs, where a single addition may use most of its bar), and each
  plausible defect of the kernels, applied to that restatement, fails them by a wide factor: a dropped leftover load, a partial loop that stops
  one CTA short, a block sum of squares without its last warp, a float4 norm without its scalar tail, a target bound of j <= tgt_n, statistics
  that ignore stats_accumulate, a slice combine without slice 15, pb rounded to 64."""
import math

import numpy as np
import pytest
import torch

from tests import tail_ref as tr

F = np.float32


# ---- tail_ref against torch ------------------------------------------------------------------------------------------------------------------------
def _torch_opt(name, params, lr):
    d, c = tr.DEFAULTS[name], tr.step_consts(name, lr, 1)
    if name in ("Adam", "AdamW"):   # the betas the kernels use: float32
        kw = dict(betas=(c["beta1"], c["beta2"]), eps=d["eps"])
        if name == "AdamW":
            kw["weight_decay"] = d["weight_decay"]
        return getattr(torch.optim, name)(params, lr=tr.f32(lr), **kw)
    if name == "RMSprop":
        return torch.optim.RMSprop(params, lr=tr.f32(lr), alpha=d["alpha"], eps=d["eps"])
    if name == "Adagrad":
        return torch.optim.Adagrad(params, lr=tr.f32(lr), eps=d["eps"])
    return torch.optim.SGD(params, lr=tr.f32(lr))


@pytest.mark.parametrize("name", tr.OPTS)
@pytest.mark.parametrize("max_norm", [0.0, 0.5, 1e3])
def test_reference_step_is_torch_optim(name, max_norm):
    """Five steps of tail_ref (step_ref with the exact clip) against torch.optim.<name> after clip_grad_norm_, in float64.  The bar, 1e-6 of the
    update plus 1e-7 of theta, is the float32 rounding of the step's constants (bias corrections, AdamW's decay), which tail_ref rounds as the
    kernels do and torch does not."""
    rng = np.random.default_rng(3)
    n, lr = 1000, 3e-3
    theta = rng.standard_normal(n)
    p = torch.nn.Parameter(torch.tensor(theta))
    opt = _torch_opt(name, [p], lr)
    m, v = np.zeros(n), np.zeros(n)
    for step in range(1, 6):
        grad_sum = rng.standard_normal(n) * 40
        stats = np.array([1.0, 37.0, 0.0, 0.0])
        ref = tr.step_ref(grad_sum, stats, theta, m, v, np.zeros(0), name, lr, max_norm, step, (0, 0, 0), 0.0)
        p.grad = torch.tensor(grad_sum / stats[1])
        before = p.detach().clone()
        if max_norm > 0:
            total = float(torch.nn.utils.clip_grad_norm_([p], max_norm))
            assert abs(total - ref["norm"]) <= 1e-12 * total
            got_clip = float((p.grad / torch.tensor(grad_sum / stats[1])).mean())
            assert abs(got_clip - ref["clip"]) <= 1e-12, (got_clip, ref["clip"])
        opt.step()
        got = p.detach().numpy()
        upd = np.abs(got - before.numpy())
        assert (np.abs(got - ref["theta"]) <= 1e-6 * upd + 1e-7 * np.abs(got) + 1e-300).all(), (name, step, float(np.abs(got - ref["theta"]).max()))
        names = {"Adam": ("exp_avg", "exp_avg_sq"), "AdamW": ("exp_avg", "exp_avg_sq"), "RMSprop": (None, "square_avg"), "Adagrad": (None, "sum"),
                 "SGD": (None, None)}[name]
        for mine, key in ((ref["m"], names[0]), (ref["v"], names[1])):
            if key:
                want = opt.state[p][key].numpy()
                assert np.allclose(mine, want, rtol=1e-6, atol=0), (name, key)
        theta, m, v = ref["theta"], ref["m"], ref["v"]


def test_step_consts_round_as_set_step_consts():
    c = tr.step_consts("Adam", 3e-4, 7)
    b1, b2 = float(F(0.9)), float(F(0.999))
    assert c["bc1"] == float(F(1 - b1 ** 7)) and c["bc2_sqrt"] == float(F(math.sqrt(1 - b2 ** 7)))
    assert tr.step_consts("RMSprop", 1e-3, 1)["beta1"] == float(F(1 - 0.99))
    assert tr.step_consts("AdamW", 1e-3, 1)["decay"] == float(F(1 - float(F(1e-3)) * 0.01))


# ---- the cases -------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_sm", [114, 132])
def test_every_case_reaches_its_edges(n_sm):
    cs = tr.cases(n_sm, n_sm)
    assert len({c.name for c in cs}) == len(cs)
    union = set()
    for c in cs:
        got = tr.reaches(c, n_sm)
        assert c.claims <= got, (c.name, sorted(c.claims - got))
        assert sum(c.ctas) <= n_sm and c.pitch >= c.P and len(c.ctas) <= 32
        mode, begin, count = c.target
        assert 0 <= begin and begin + count <= c.n
        union |= got
    missing = tr.needed(n_sm) - union
    print(f"{n_sm} SMs: {len(cs)} cases, {len(union)} edges")
    assert not missing, sorted(missing)


def test_shape_switches():
    C = 132
    assert tr.tail_shape(C * 96, C) is None and tr.tail_shape(C * 96 + 1, C) == (128, 4)
    assert tr.tail_shape(C * 256, C) == (256, 4) and tr.tail_shape(C * 256 + 1, C) == (288, 3)
    assert tr.tail_shape(C * 320, C) == (320, 3) and tr.tail_shape(C * 320 + 1, C) == (352, 2)
    assert tr.tail_shape(C * 512, C) == (512, 2) and tr.tail_shape(C * 512 + 1, C) is None
    assert tr.tail_shape(38668, 114) == (352, 2) and tr.tail_shape(38668, 132) == (320, 3)   # the default two-agent LBF learner


# ---- float32 restatement in the kernels' order -----------------------------------------------------------------------------------------------------
def _butterfly(x):
    """__shfl_xor_sync tree over the last axis (32 lanes): lane 0's result"""
    x = x.copy()
    for off in (16, 8, 4, 2, 1):
        x = x + x[..., np.arange(32) ^ off]
    return x[..., 0]


def reduce16(scratch, ctas, P, drop_t2=False, drop_slice15=False):
    """grad_reduce_kernel's sums: slice q takes CTAs q, q + 16, ... four at a time, then up to three leftovers; the slices combine four by four"""
    out = []
    for c0, cnt in zip(tr.cta_begin(ctas), ctas):
        X = scratch[c0:c0 + cnt, :P]
        z = np.zeros(P, F)
        part = []
        for q in range(16):
            a = [z.copy() for _ in range(4)]
            c = q
            while c + 48 < cnt:
                for k in range(4):
                    a[k] = a[k] + X[c + 16 * k]
                c += 64
            t = [X[c + 16 * k] if c + 16 * k < cnt and not (k == 2 and drop_t2) else z for k in range(3)]
            part.append(((a[0] + a[1]) + (a[2] + a[3])) + ((t[0] + t[1]) + t[2]))
        if drop_slice15:
            part[15] = z
        g = z.copy()
        for k in range(0, 16, 4):
            g = g + ((part[k] + part[k + 1]) + (part[k + 2] + part[k + 3]))
        out.append(g)
    return np.concatenate(out)


def reduce_fused(scratch, ctas, P, ns, short=False):
    """reduce_adam_kernel's sums: slice q takes CTAs q, q + ns, ... in rounds of 20 loads, fives summed in pairs; then the slices in order"""
    out = []
    for c0, cnt in zip(tr.cta_begin(ctas), ctas):
        X = scratch[c0:c0 + cnt, :P]
        z = np.zeros(P, F)
        end = cnt - 1 if short else cnt
        part = []
        for q in range(ns):
            s = z.copy()
            for cb in range(q, cnt, 20 * ns):
                v = [X[cb + k * ns] if cb + k * ns < end else z for k in range(20)]
                u = [(v[4 * k] + v[4 * k + 1]) + (v[4 * k + 2] + v[4 * k + 3]) for k in range(5)]
                s = s + (((u[0] + u[1]) + (u[2] + u[3])) + u[4])
            part.append(s)
        g = part[0]
        for k in range(1, ns):
            g = g + part[k]
        out.append(g)
    return np.concatenate(out)


def stats_f32(loss_part, n_parts, stats_in, accumulate, ignore_accumulate=False):
    x = np.zeros((4, 32 * max(1, -(-n_parts // 32))), F)
    x[:, :n_parts] = loss_part[:n_parts].T
    lanes = np.zeros((4, 32), F)
    for r in range(x.shape[1] // 32):
        lanes = lanes + x[:, 32 * r:32 * r + 32]
    t = _butterfly(lanes)
    return (stats_in.astype(F) if accumulate and not ignore_accumulate else np.zeros(4, F)) + t


def norm_f32(grad, fill, path, shape, skip_last_warp=False, skip_tail=False):
    n = len(grad)
    inv = F(1) / F(fill)
    if path == 0:
        pb = shape[0]
        grid = -(-n // pb)
        g = np.zeros(grid * pb, F); g[:n] = grad
        w = _butterfly((g * g).reshape(grid, pb // 32, 32))   # [grid][warps]
        x = w[:, 0].copy()
        for k in range(1, pb // 32 - (1 if skip_last_warp else 0)):
            x = x + w[:, k]
        lanes = np.zeros(32, F)
        for r in range(-(-grid // 32)):
            blk = np.zeros(32, F); seg = x[32 * r:32 * r + 32]; blk[:len(seg)] = seg
            lanes = lanes + blk
        return F(np.sqrt(_butterfly(lanes))) * inv
    red = np.zeros(256, F)
    if path == 1:
        nb = -(-n // 64)
        g = np.zeros(nb * 64, F); g[:n] = grad
        sq = (g * g).reshape(nb, 64)
        part = _butterfly(sq[:, :32] + sq[:, 32:])
        for r in range(-(-nb // 256)):
            blk = np.zeros(256, F); seg = part[256 * r:256 * r + 256]; blk[:len(seg)] = seg
            red = red + blk
    else:
        n4 = n // 4
        a = (grad[:4 * n4] * inv).reshape(n4, 4).astype(np.float64)
        for r in range(-(-n4 // 256)):
            rows = a[256 * r:256 * r + 256]
            for k in range(4):
                blk = np.zeros(256); blk[:len(rows)] = rows[:, k]
                red = (blk * blk + red.astype(np.float64)).astype(F)   # fmaf(a, a, s): the product is exact in double
        if not skip_tail:
            for i in range(4 * n4, n):
                t = i - 4 * n4
                gi = np.float64(grad[i] * inv)
                red[t] = F(gi * gi + np.float64(red[t]))
    k = 128
    while k:
        red[:k] = red[:k] + red[k:2 * k]
        k //= 2
    return F(np.sqrt(red[0])) * (inv if path == 1 else F(1))


def step_f32(opt, c, g, m, v, th):
    g, m, v, th = (np.asarray(x, F) for x in (g, m, v, th))
    k = {key: F(val) for key, val in c.items()}
    if opt in ("Adam", "AdamW"):
        th = th * k["decay"] if opt == "AdamW" else th
        m = m + (g - m) * (F(1) - k["beta1"])
        v = v * k["beta2"] + g * g * (F(1) - k["beta2"])
        denom = np.sqrt(v) / k["bc2_sqrt"] + k["eps"]
        return th - (k["lr"] / k["bc1"]) * (m / denom), m, v
    if opt in ("RMSprop", "Adagrad"):
        v = (k["beta1"] * g) * g + v * k["beta2"] if opt == "RMSprop" else g * g + v
        return th + (-k["lr"] * g) / (np.sqrt(v) + k["eps"]), m, v
    return th - k["lr"] * g, m, v


def tail_f32(case, path, opt, scratch, lp, stats_in, theta, m, v, tgt, grad_clip, lr=3e-4, tau=0.05, defect=None):
    """the tail of one case in float32 in the kernels' order -> (grad, stats, theta, m, v, tgt with GUARD words each side, loss_out, shape)"""
    n = case.n
    shape = tr.tail_shape(n, 132) if defect != "pb rounded to 64" else _shape64(n, 132)
    if path == 0:
        grad = reduce_fused(scratch, case.ctas, case.P, shape[1], short=defect == "partial loop one CTA short")
    else:
        grad = reduce16(scratch, case.ctas, case.P, drop_t2=defect == "third leftover load dropped", drop_slice15=defect == "slice 15 not combined")
    stats = stats_f32(lp, case.n_loss_parts, stats_in, case.accumulate, ignore_accumulate=defect == "stats_accumulate ignored" and path != 0)
    fill = stats[1]
    norm = norm_f32(grad, fill, path, shape, skip_last_warp=defect == "block sum of squares without its last warp" and path == 0,
                    skip_tail=defect == "float4 norm without its scalar tail" and path == 2)
    clip = tr.device_clip(norm, grad_clip)
    g = (grad * (F(1) / F(fill))) * clip
    th, m2, v2 = step_f32(opt, tr.step_consts(opt, lr, case.step), g, m, v, theta)
    mode, begin, count = case.target
    G = 8
    t = np.full(count + 2 * G, F(4242.0)); t[G:G + count] = tgt
    hi = count + 1 if defect == "target bound j <= tgt_n" else count
    for j in range(min(hi, n - begin)):
        if mode == 1:
            t[G + j] = th[begin + j]
        elif mode == 2:
            t[G + j] = (F(1) - F(tau)) * t[G + j] + F(tau) * th[begin + j]
    loss_out = np.array([stats[0] * (F(1) / fill), norm, stats[2] * (F(1) / fill), stats[3] * (F(1) / fill), fill, 0], F)
    return grad, stats, th, m2, v2, t, loss_out, shape


def _shape64(n, capacity):
    pb = (-(-n // capacity) + 63) // 64 * 64
    if pb < 128 or pb > 512:
        return None
    return pb, min(1024 // pb, 4)


def bar_fractions(case, path, opt, out, scratch, lp, stats_in, theta, m, v, tgt, grad_clip, kind):
    """each check of the GPU test on the outputs `out` of a tail: {check: fraction of its bar} (inf: an exact check or a sentinel failed)"""
    grad, stats, th, m2, v2, t, loss_out, shape = out
    n = case.n
    r = {}
    ref_g, ref_s = tr.reduce_ref(scratch, case.ctas, case.P, lp, case.n_loss_parts, stats_in, case.accumulate)
    if shape != tr.tail_shape(n, 132):
        r["shape"] = np.inf
    if kind == "int":
        r["integer sums"] = 0.0 if np.array_equal(grad, ref_g.astype(F)) and np.array_equal(stats, ref_s.astype(F)) else np.inf
        return r
    gbar = np.concatenate([(c + 2) * tr.U * np.abs(scratch[s:s + c, :case.P]).astype(np.float64).sum(0) for s, c in zip(tr.cta_begin(case.ctas), case.ctas)])
    sbar = (case.n_loss_parts + 3) * tr.U * (np.abs(lp[:case.n_loss_parts]).astype(np.float64).sum(0) + (np.abs(stats_in) if case.accumulate else 0))
    r["gradient"] = tr.worst(grad, ref_g, gbar)
    r["statistics"] = tr.worst(stats, ref_s, sbar)
    gd, sd = grad.astype(np.float64), stats.astype(np.float64)
    norm_d = math.sqrt(float((gd * gd).sum())) / sd[1]
    nb = tr.norm_bar(path, n, tr.tail_shape(n, 132))
    r["norm"] = abs(float(loss_out[1]) - norm_d) / (nb * norm_d)
    dclip = tr.device_clip(loss_out[1], grad_clip)
    r["clip"] = abs(float(dclip) - tr.clip_coef(norm_d, grad_clip)) / ((nb + 3 * tr.U) * tr.clip_coef(norm_d, grad_clip))
    ref = tr.step_ref(gd, sd, theta, m, v, tgt, opt, 3e-4, grad_clip, case.step, case.target, 0.05, clip=dclip)
    bars = tr.step_bars(opt, ref, theta, tgt, 0.05, case.target)
    r["theta"] = tr.worst(th, ref["theta"], bars["theta"])
    if opt in tr.USES_M:
        r["m"] = tr.worst(m2, ref["m"], bars["m"])
    if opt in tr.USES_V:
        r["v"] = tr.worst(v2, ref["v"], bars["v"])
    mode, begin, count = case.target
    G = 8
    if (t[:G] != 4242.0).any() or (t[G + count:] != 4242.0).any():
        r["target sentinels"] = np.inf
    if mode == 1:
        r["hard target"] = 0.0 if np.array_equal(t[G:G + count], th[begin:begin + count]) else np.inf
    elif mode == 2:
        r["Polyak target"] = tr.worst(t[G:G + count], ref["tgt"][:count], bars["tgt"])
    return r


def _inputs(case, kind, seed):
    rng = np.random.default_rng(seed)
    rows = sum(case.ctas)
    if kind == "int":
        scratch = rng.integers(-8, 9, size=(rows, case.P)).astype(F)
        lp = rng.integers(-8, 9, size=(case.n_loss_parts, 4)).astype(F)
        stats_in = np.array([3, 5, -2, 7], F)
    else:
        scratch = ((1e3 if case.clip == "off" else 1.0) * rng.standard_normal((rows, case.P))).astype(F)
        lp = rng.standard_normal((case.n_loss_parts, 4)).astype(F)
        stats_in = np.array([0.25, 3.0, -1.5, 2.0], F)
    lp[:, 1] = rng.integers(1, 5, size=case.n_loss_parts)
    n = case.n
    theta = (0.1 * rng.standard_normal(n)).astype(F)
    m = (1e-3 * rng.standard_normal(n)).astype(F) if case.step > 1 else np.zeros(n, F)
    v = (1e-6 * np.abs(rng.standard_normal(n))).astype(F) if case.step > 1 else np.zeros(n, F)
    tgt = (0.1 * rng.standard_normal(case.target[2])).astype(F)
    ref_g, ref_s = tr.reduce_ref(scratch, case.ctas, case.P, lp, case.n_loss_parts, stats_in, case.accumulate)
    norm = math.sqrt(float((ref_g ** 2).sum())) / ref_s[1]
    grad_clip = tr.f32({"off": 0.0, "below": norm * (1 - 2 ** -10), "above": norm * (1 + 2 ** -10), "active": norm / 100, "mild": 2 * norm}[case.clip])
    return scratch, lp, stats_in, theta, m, v, tgt, grad_clip


SAMPLE = ("pb128_low", "pb256_top", "pb288_low", "pb352_top-1", "pb512_top", "small_n1", "small_n5", "small_n65", "small_n257", "one_net_C_ctas",
          "nets_16_17_15_48", "nets_39_41_47_3", "nets_63_64_5_p18", "nets_81_2_1")


def _sample_cases():
    by = {c.name: c for c in tr.cases(132, 132)}
    return [by[k] for k in SAMPLE]


@pytest.mark.parametrize("name", SAMPLE)
def test_float32_restatement_passes_the_bars_with_margin(name):
    case = {c.name: c for c in tr.cases(132, 132)}[name]
    for path in case.paths:
        if path == 0 and tr.tail_shape(case.n, 132) is None:
            continue
        for opt in tr.OPTS:
            for kind in ("int", "gauss"):
                args = _inputs(case, kind, 11)
                out = tail_f32(case, path, opt, *args)
                fr = bar_fractions(case, path, opt, out, *args, kind=kind)
                w = max(fr.values())
                print(f"{name} path {path} {opt} {kind}: worst {w:.3f} of the bar ({max(fr, key=fr.get)})")
                assert w <= 1 / 2, (name, path, opt, kind, max(fr, key=fr.get), w)


DEFECTS = {   # defect -> (paths it applies to, the checks it must fail)
    "third leftover load dropped": ((1, 2), ("integer sums", "gradient")),
    "partial loop one CTA short": ((0,), ("integer sums", "gradient")),
    "block sum of squares without its last warp": ((0,), ("norm",)),
    "float4 norm without its scalar tail": ((2,), ("norm",)),
    "target bound j <= tgt_n": ((0, 1, 2), ("target sentinels",)),
    "stats_accumulate ignored": ((1, 2), ("integer sums", "statistics")),
    "slice 15 not combined": ((1, 2), ("integer sums", "gradient")),
    "pb rounded to 64": ((0,), ("shape",)),
}


@pytest.mark.parametrize("defect", list(DEFECTS))
def test_defects_fail_the_bars(defect):
    """each defect fails every check it should on at least one sampled case, by 100x or more where the bar is a tolerance"""
    paths, checks = DEFECTS[defect]
    failed = {k: 0.0 for k in checks}
    for case in _sample_cases():
        for path in paths:
            if path not in case.paths or (path == 0 and tr.tail_shape(case.n, 132) is None):
                continue
            for kind in ("int", "gauss"):
                args = _inputs(case, kind, 11)
                opt = "Adam"
                try:
                    out = tail_f32(case, path, opt, *args, defect=defect)
                except TypeError:   # pb rounded to 64 may leave no shape: the refusal itself is the failure
                    failed["shape"] = np.inf
                    continue
                fr = bar_fractions(case, path, opt, out, *args, kind=kind)
                for k in checks:
                    failed[k] = max(failed[k], fr.get(k, 0.0))
    print(f"{defect}: " + ", ".join(f"{k} at {v:.3g}x its bar" for k, v in failed.items()))
    for k, v in failed.items():
        assert v >= 100, (defect, k, v)


@pytest.mark.parametrize("n_sm", [114, 132])
def test_learner_finder_reaches_every_fused_class(n_sm):
    """the IDQN configurations of the GPU test's learner-level cases: one in every pb class, a class of H = 128 (the tensor-core images) among
    them, n = C * 96 + 1 or the nearest above it, and the nearest n on each side of both refusals"""
    cs = tr.learner_cases(n_sm)
    for pb in range(tr.MIN_PB, tr.MAX_PB + 1, 32):
        N, D, H, A, n = cs[f"pb={pb}"]
        assert tr.dqn_params(N, D, H, A) == n and tr.tail_shape(n, n_sm)[0] == pb and N <= 4 and D <= 31
    assert any(c[2] == 128 for c in cs.values())
    assert tr.tail_shape(cs["pb=128 small edge"][4], n_sm) == (128, 4) and tr.tail_shape(cs["refused below"][4], n_sm) is None
    assert tr.tail_shape(cs["pb=512 top"][4], n_sm) == (512, 2) and tr.tail_shape(cs["refused above"][4], n_sm) is None
    assert cs["refused below"][4] <= n_sm * 96 < cs["pb=128 small edge"][4] and cs["pb=512 top"][4] <= n_sm * 512 < cs["refused above"][4]
    if n_sm == 132:
        assert cs["pb=128 small edge"][4] == n_sm * 96 + 1 and cs["refused below"][4] == n_sm * 96


def test_ia2c_configurations_cover_the_scalar_tail():
    for A, rem in ((4, 1), (5, 2), (6, 3)):
        na, nc = tr.ac_params(1, 10, 128, A)
        assert (na + nc) % 4 == rem
    assert tr.ac_params(1, 10, 128, 5)[0] % 2 == 1

"""GPU: the update tail (reduction of the per-CTA gradient partials, loss statistics, clip_grad_norm_, the optimiser step, the target update) alone,
through marl_debug_tail_run, at every case tests/tail_ref.py generates for this device's capacity C -- every fused block shape pb x ns, both
refusals, the per-network CTA counts at the edges of both reductions -- on each path the case allows (0 fused, 1 two kernels with the per-block
sums of squares, 2 without them), against the float64 reference.

Bars (derived, not measured; u = 2^-24):
- integer partials in [-8, 8] (integer loss statistics): every partial sum is an integer below 2^24, so float32 adds them exactly in any order:
  grad[0..n) and the four statistics must equal the float64 sums bit for bit -- a dropped, repeated or misattributed partial is an exact failure.
- Gaussian partials: a sum of k terms in any bracketing is within (k - 1) u sum|terms| of the exact sum (first order), so each reduced gradient
  is within (n_cta + 2) u sum_c |partial_c| of float64 (n_cta: its network's CTAs; + 2 for slack, as one addition may use its full unit), each
  statistic within (n_loss_parts + 3) u sum |parts| (+ its carried value when accumulating); and two launches are bit-identical (the combine is
  in a fixed order).
- the norm (loss_out[1]) against sqrt(sum g^2) / fill of the device's own gradient in float64: relative (L + 8) u, L the longest chain of
  additions of the path's sum of squares (tail_ref.norm_chain); the clip coefficient the kernels form from it against clip_grad_norm_'s exact
  one: that relative bar plus 3 u (the division, the + 1e-6 and min).
- the step from the device's gradient and its own clip coefficient (g = (grad * (1 / fill)) * clip in float32 is then the kernels' exact g):
  tail_ref.step_bars, a few u of each term's no-cancellation scale; a hard-copied target is bit-equal to the new theta; loss_out[0, 2, 3]
  within 3 u of stats / fill (1 / fill and the product round), loss_out[4] equal to fill.
- sentinels: NaN in the scratch padding [P, pitch), in the scratch rows past the last CTA and in loss_part past n_loss_parts (a read of any
  makes a result NaN); guard words after grad[n + 4], theta, m, v and the sums of squares, around theta_tgt's slice; the m / v buffer an
  optimiser does not use -- all must come back untouched.
- the shape marl_debug_tail_shape reports equals tail_ref.tail_shape for every case; path 0 returns MARL_EINVAL at both refusals and launches
  nothing (every buffer comes back as it went in).
Learner level (test_idqn_handle_tail, test_ia2c_handle_tail): IDQN handles whose parameter count tail_ref.learner_cases puts in every fused class
this device reaches and on each side of both refusals, and IA2C at n % 4 = 1, 2, 3 with hard and Polyak targets -- the learners' own reduction and
step parameters (sums-of-squares buffer, grads_are_local, tensor-core images, the critic-only target slice) against the oracle's gradient (1e-5)
and tail_ref's step from the device's gradient (the bars above).
Run with -s to see each check's worst error as a fraction of its bar."""
import copy
import ctypes as C
import math
import os
import re

import numpy as np
import pytest
import torch

from tests import tail_ref as tr

pytestmark = pytest.mark.gpu
GUARD = 8
EINVAL = -1
OPT_KIND = {name: k for k, name in enumerate(tr.OPTS)}


def _max_agents():
    """MARL_MAX_AGENTS from the header: the length of marl_debug_tail.cta_begin is MARL_MAX_AGENTS + 1"""
    with open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "marl_b200.h")) as f:
        return int(re.search(r"^#define MARL_MAX_AGENTS (\d+)", f.read(), re.M).group(1))


class Tail(C.Structure):
    _fields_ = [("n_nets", C.c_int32), ("P", C.c_int32), ("scratch_pitch", C.c_int32), ("cta_begin", C.c_int32 * (_max_agents() + 1)),
                ("scratch", C.c_void_p), ("loss_part", C.c_void_p), ("n_loss_parts", C.c_int32), ("stats_accumulate", C.c_int32),
                ("grad", C.c_void_p), ("sumsq", C.c_void_p), ("theta", C.c_void_p), ("theta_tgt", C.c_void_p), ("m", C.c_void_p), ("v", C.c_void_p),
                ("tgt_begin", C.c_int32), ("tgt_n", C.c_int32), ("target_mode", C.c_int32), ("tau", C.c_float),
                ("lr", C.c_float), ("grad_clip", C.c_float), ("step", C.c_int64), ("loss_out", C.c_void_p)]


def _lib():
    from codebase_b200 import _native as nat

    return nat.lib()


def _optimizer(name):
    from codebase_b200 import _native as nat

    d = tr.DEFAULTS[name]
    return nat.Optimizer(OPT_KIND[name], d.get("beta1", 0.0), d.get("beta2", 0.0), d.get("alpha", 0.0), d.get("eps", 0.0), d.get("weight_decay", 0.0))


def device_shape(n, opt="Adam"):
    """(rc, (pb, ns), capacity) from marl_debug_tail_shape"""
    pb, ns, cap = C.c_int32(), C.c_int32(), C.c_int32()
    rc = _lib().marl_debug_tail_shape(C.c_int32(n), C.c_int32(OPT_KIND[opt]), C.c_int32(torch.cuda.current_device()), C.byref(pb), C.byref(ns), C.byref(cap))
    return rc, (pb.value, ns.value), cap.value


def _device():
    n_sm = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    _, _, cap = device_shape(1)
    assert cap >= n_sm, (cap, n_sm)
    return n_sm, cap


# ---- one case's buffers ----------------------------------------------------------------------------------------------------------------------------
class Buffers:
    """Device buffers of one case with their sentinels; `fresh` resets everything a launch may write."""

    def __init__(self, case, rng):
        n, dev = case.n, "cuda"
        self.case = case
        rows = sum(case.ctas)
        self.scratch = torch.full((rows + 2, case.pitch), float("nan"), device=dev)
        self.loss_part = torch.full((case.n_loss_parts + 2, 4), float("nan"), device=dev)
        self.grad = torch.empty(n + 4 + GUARD, device=dev)
        self.n_sumsq = -(-n // 64) + 1
        self.sumsq = torch.empty(self.n_sumsq + GUARD, device=dev)
        mode, begin, count = case.target
        self.theta = torch.empty(n + GUARD, device=dev)
        self.m = torch.empty(n + GUARD, device=dev)
        self.v = torch.empty(n + GUARD, device=dev)
        self.tgt = torch.empty(count + 2 * GUARD, device=dev)
        self.loss_out = torch.empty(6 + GUARD, device=dev)
        self.theta0 = (0.1 * rng.standard_normal(n)).astype(np.float32)
        self.tgt0 = (0.1 * rng.standard_normal(count)).astype(np.float32)
        if case.step > 1:
            self.m0 = (1e-3 * rng.standard_normal(n)).astype(np.float32)
            self.v0 = (1e-6 * np.abs(rng.standard_normal(n))).astype(np.float32)
        else:
            self.m0 = self.v0 = np.zeros(n, np.float32)

    def load_partials(self, scratch, loss_part):
        c = self.case
        self.scratch[: scratch.shape[0], : c.P] = torch.as_tensor(scratch)
        self.loss_part[: c.n_loss_parts] = torch.as_tensor(loss_part)

    def fresh(self, opt, stats_in):
        n = self.case.n
        self.grad.fill_(float("nan")); self.grad[n:n + 4] = torch.as_tensor(stats_in); self.grad[n + 4:] = 7777.0
        self.sumsq.fill_(-5555.0)
        self.theta[:n] = torch.as_tensor(self.theta0); self.theta[n:] = 8888.0
        for buf, init, used in ((self.m, self.m0, opt in tr.USES_M), (self.v, self.v0, opt in tr.USES_V)):
            buf.fill_(31337.0)
            if used:
                buf[:n] = torch.as_tensor(init)
        self.tgt.fill_(4242.0); self.tgt[GUARD:GUARD + len(self.tgt0)] = torch.as_tensor(self.tgt0)
        self.loss_out.fill_(-1.0)

    def run(self, opt, path, lr, grad_clip, tau=0.05):
        c = self.case
        mode, begin, count = c.target
        t = Tail()
        t.n_nets, t.P, t.scratch_pitch = len(c.ctas), c.P, c.pitch
        for k, b in enumerate(tr.cta_begin(c.ctas)):
            t.cta_begin[k] = int(b)
        t.scratch, t.loss_part = self.scratch.data_ptr(), self.loss_part.data_ptr()
        t.n_loss_parts, t.stats_accumulate = c.n_loss_parts, c.accumulate
        t.grad, t.sumsq, t.theta, t.m, t.v = (x.data_ptr() for x in (self.grad, self.sumsq, self.theta, self.m, self.v))
        t.theta_tgt = self.tgt.data_ptr() + 4 * GUARD
        t.tgt_begin, t.tgt_n, t.target_mode, t.tau = begin, count, mode, tau
        t.lr, t.grad_clip, t.step = lr, grad_clip, c.step
        t.loss_out = self.loss_out.data_ptr()
        o = _optimizer(opt)
        rc = _lib().marl_debug_tail_run(C.byref(t), C.byref(o), C.c_int32(path), C.c_int32(torch.cuda.current_device()),
                                        C.c_void_p(torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        return rc

    def state(self):
        return {k: getattr(self, k).cpu().numpy().copy() for k in ("grad", "sumsq", "theta", "m", "v", "tgt", "loss_out")}


# ---- the checks ------------------------------------------------------------------------------------------------------------------------------------
WORST = {}   # check -> (fraction of its bar, where)


def _record(check, ratio, where):
    if ratio > WORST.get(check, (-1.0, ""))[0]:
        WORST[check] = (ratio, where)


def _note(check, ratio, where):
    _record(check, ratio, where)
    assert ratio <= 1.0, f"{where}: {check} at {ratio:.3g} x its bar"


def _record_grad(got, want, where):
    """the gradient against the oracle as a fraction of assert_grad_close's bar, 1e-5 x max(1, max |want|) (which it then asserts)"""
    want = np.asarray(want, np.float64)
    _record("learner: gradient vs oracle", float(np.abs(np.asarray(got, np.float64) - want).max()) / (1e-5 * max(1.0, float(np.abs(want).max()))), where)


def _partials(case, rng, kind):
    rows = sum(case.ctas)
    if kind == "int":
        scratch = rng.integers(-8, 9, size=(rows, case.P)).astype(np.float32)
        lp = rng.integers(-8, 9, size=(case.n_loss_parts, 4)).astype(np.float32)
        lp[:, 1] = rng.integers(1, 5, size=case.n_loss_parts)
        stats_in = np.array([3, 5, -2, 7], np.float32)
    else:
        scale = 1e3 if case.clip == "off" else 1.0
        scratch = (scale * rng.standard_normal((rows, case.P))).astype(np.float32)
        lp = rng.standard_normal((case.n_loss_parts, 4)).astype(np.float32)
        lp[:, 1] = rng.integers(1, 5, size=case.n_loss_parts)
        stats_in = np.array([0.25, 3.0, -1.5, 2.0], np.float32)
    return scratch, lp, stats_in


def _grad_clip(case, norm):
    return {"off": 0.0, "below": norm * (1 - 2 ** -10), "above": norm * (1 + 2 ** -10), "active": norm / 100, "mild": 2 * norm}[case.clip]


def _check_sentinels(case, b, s, path, opt, where):
    n = case.n
    mode, begin, count = case.target
    assert (s["grad"][n + 4:] == 7777.0).all(), f"{where}: guard words after grad[n + 4] written"
    assert (s["theta"][n:] == 8888.0).all(), f"{where}: guard words after theta written"
    for name, used in (("m", opt in tr.USES_M), ("v", opt in tr.USES_V)):
        tail = s[name][n:] if used else s[name]
        assert (tail == 31337.0).all(), f"{where}: {name} written {'past n' if used else 'though ' + opt + ' keeps no ' + name}"
    assert (s["tgt"][:GUARD] == 4242.0).all() and (s["tgt"][GUARD + count:] == 4242.0).all(), f"{where}: theta_tgt written outside its slice"
    if mode == 0:
        assert np.array_equal(s["tgt"][GUARD:GUARD + count], b.tgt0), f"{where}: target mode 0 changed theta_tgt"
    first_free = {0: -(-n // (tr.tail_shape(n, CAP[1]) or (1, 0))[0]) if path == 0 else 0, 1: -(-n // 64), 2: 0}[path]
    assert (s["sumsq"][first_free:] == -5555.0).all(), f"{where}: sums of squares written past block {first_free}"
    assert (s["loss_out"][6:] == -1.0).all(), f"{where}: loss_out written past [6]"


def run_case(case, rng):
    n, P = case.n, case.P
    b = Buffers(case, rng)
    shape = tr.tail_shape(n, CAP[1])
    rc, dshape, _ = device_shape(n)
    assert (rc == 0) == (shape is not None) and (shape is None or dshape == shape), f"{case.name}: device shape {rc, dshape} != {shape}"
    iscratch, ilp, istats = _partials(case, rng, "int")
    gscratch, glp, gstats = _partials(case, rng, "gauss")
    iref = tr.reduce_ref(iscratch, case.ctas, P, ilp, case.n_loss_parts, istats, case.accumulate)
    gref = tr.reduce_ref(gscratch, case.ctas, P, glp, case.n_loss_parts, gstats, case.accumulate)
    gbar = np.concatenate([(c + 2) * tr.U * np.abs(gscratch[s:s + c]).astype(np.float64).sum(0) for s, c in zip(tr.cta_begin(case.ctas), case.ctas)])
    sbar = (case.n_loss_parts + 3) * tr.U * (np.abs(glp).astype(np.float64).sum(0) + (np.abs(gstats) if case.accumulate else 0))
    norm64 = math.sqrt(float((gref[0] ** 2).sum())) / gref[1][1]
    grad_clip = tr.f32(_grad_clip(case, norm64))
    lr = 3e-4
    for path in case.paths:
        for opt in case.opts:
            where = f"{case.name} path {path} {opt}"
            if path == 0 and shape is None:   # the refusal: nothing launches
                b.load_partials(gscratch, glp); b.fresh(opt, gstats)
                before = b.state()
                assert b.run(opt, 0, lr, grad_clip) == EINVAL, f"{where}: the fused tail accepted a shape reduce_adam_shape refuses"
                after = b.state()
                for k in before:
                    assert np.array_equal(before[k], after[k], equal_nan=True), f"{where}: refused, but {k} changed"
                continue
            # integer partials: exact
            b.load_partials(iscratch, ilp); b.fresh(opt, istats)
            assert b.run(opt, path, lr, 0.0) == 0, where
            s = b.state()
            assert np.array_equal(s["grad"][:n], iref[0].astype(np.float32)), \
                f"{where}: integer partials: {int((s['grad'][:n] != iref[0]).sum())} gradient sums differ, first at {int(np.argmax(s['grad'][:n] != iref[0]))}"
            assert np.array_equal(s["grad"][n:n + 4], iref[1].astype(np.float32)), f"{where}: integer statistics {s['grad'][n:n + 4]} != {iref[1]}"
            _check_sentinels(case, b, s, path, opt, where + " (integer)")
            # Gaussian partials: twice, bit-identical
            runs = []
            for _ in range(2):
                b.load_partials(gscratch, glp); b.fresh(opt, gstats)
                assert b.run(opt, path, lr, grad_clip) == 0, where
                runs.append(b.state())
            s = runs[0]
            for k in s:
                assert np.array_equal(s[k], runs[1][k], equal_nan=True), f"{where}: two launches differ in {k}"
            _check_sentinels(case, b, s, path, opt, where)
            _note("reduced gradient (Gaussian)", tr.worst(s["grad"][:n], gref[0], gbar), where)
            _note("statistics (Gaussian)", tr.worst(s["grad"][n:n + 4], gref[1], sbar), where)
            gd, sd = s["grad"][:n].astype(np.float64), s["grad"][n:n + 4].astype(np.float64)
            fill = sd[1]
            norm_d = math.sqrt(float((gd * gd).sum())) / fill
            nb = tr.norm_bar(path, n, shape)
            _note("norm", abs(float(s["loss_out"][1]) - norm_d) / (nb * norm_d), where)
            dclip = tr.device_clip(s["loss_out"][1], grad_clip)
            exact = tr.clip_coef(norm_d, grad_clip)
            _note("clip coefficient", abs(float(dclip) - exact) / ((nb + 3 * tr.U) * exact), where)
            if case.clip == "above":
                assert dclip == 1.0, f"{where}: clipped a norm below the clip"
            if case.clip in ("below", "active"):
                assert dclip < 1.0, f"{where}: did not clip"
            ref = tr.step_ref(gd, sd, b.theta0, b.m0, b.v0, b.tgt0, opt, lr, grad_clip, case.step, case.target, 0.05, clip=dclip)
            bars = tr.step_bars(opt, ref, b.theta0, b.tgt0, 0.05, case.target)
            _note(f"theta ({opt})", tr.worst(s["theta"][:n], ref["theta"], bars["theta"]), where)
            if opt in tr.USES_M:
                _note("m", tr.worst(s["m"][:n], ref["m"], bars["m"]), where)
            if opt in tr.USES_V:
                _note(f"v ({opt})", tr.worst(s["v"][:n], ref["v"], bars["v"]), where)
            mode, begin, count = case.target
            tgt = s["tgt"][GUARD:GUARD + count]
            if mode == 1:
                assert np.array_equal(tgt, s["theta"][begin:begin + count]), f"{where}: hard target is not the new theta"
            elif mode == 2:
                _note("Polyak target", tr.worst(tgt, ref["tgt"][:count], bars["tgt"]), where)
            lo = s["loss_out"][:6].astype(np.float64)
            for k in (0, 2, 3):
                _note("loss_out", abs(lo[k] - sd[k] / fill) / max(3 * tr.U * abs(sd[k] / fill), 1e-38), where)
            assert lo[4] == np.float32(fill) and lo[5] == 0.0, f"{where}: loss_out {lo}"


CAP = []


@pytest.fixture(scope="module", autouse=True)
def _capacity():
    CAP[:] = list(_device())
    yield
    print("\nworst error of each check, as a fraction of its bar (device: %s, %d SMs, capacity %d):" % (torch.cuda.get_device_name(), CAP[0], CAP[1]))
    for k, (r, where) in sorted(WORST.items()):
        print(f"  {k:28s} {r:.3g}   ({where})")


GROUPS = ("pb", "refuse", "small", "largest", "nets", "one_net")


@pytest.mark.parametrize("group", GROUPS)
def test_tail_matches_float64(group):
    todo = [c for c in tr.cases(*CAP) if c.name.startswith(group)]
    assert todo, group
    for i, case in enumerate(todo):
        run_case(case, np.random.default_rng(1000 * GROUPS.index(group) + i))


def test_every_case_reaches_its_edges_on_this_device():
    cs = tr.cases(*CAP)
    union = set()
    for c in cs:
        got = tr.reaches(c, CAP[1])
        assert c.claims <= got, (c.name, c.claims - got)
        union |= got
    assert tr.needed(CAP[1]) <= union, tr.needed(CAP[1]) - union


def test_out_of_range_arguments_are_refused():
    b = Buffers(tr.Case("refusals", 100, (2,), 101, 1, 0, ("Adam",), "mild", 1, (1, 0, 100), (1,)), np.random.default_rng(0))
    lib = _lib()

    def rc(**kw):
        c = b.case
        t = Tail()
        t.n_nets, t.P, t.scratch_pitch = 1, c.P, c.pitch
        t.cta_begin[0], t.cta_begin[1] = 0, 2
        t.scratch, t.loss_part, t.n_loss_parts = b.scratch.data_ptr(), b.loss_part.data_ptr(), 1
        t.grad, t.sumsq, t.theta, t.m, t.v, t.theta_tgt = (x.data_ptr() for x in (b.grad, b.sumsq, b.theta, b.m, b.v, b.tgt))
        t.tgt_begin, t.tgt_n, t.target_mode, t.lr, t.step = 0, 100, 1, 1e-3, 1
        for k, v in kw.items():
            if k == "cta_begin":
                for i, x in enumerate(v):
                    t.cta_begin[i] = x
            else:
                setattr(t, k, v)
        o = _optimizer("Adam")
        r = lib.marl_debug_tail_run(C.byref(t), C.byref(o), C.c_int32(1), C.c_int32(torch.cuda.current_device()), None)
        torch.cuda.synchronize()
        return r, lib.marl_last_error().decode()

    for kw, words in ((dict(n_nets=33), "n_nets"), (dict(scratch_pitch=99), "scratch_pitch"), (dict(n_nets=2, cta_begin=(0, 2, 1)), "cta_begin"),
                      (dict(tgt_begin=1), "target slice"), (dict(tgt_n=101), "target slice"), (dict(target_mode=3), "target_mode"),
                      (dict(step=0), "step"), (dict(stats_accumulate=2), "stats_accumulate"), (dict(grad=b.grad.data_ptr() + 4), "aligned")):
        r, msg = rc(**kw)
        assert r == EINVAL and words in msg, (kw, r, msg)


# ---- learner level: real handles at every fused class this device reaches ----------------------------------------------------------------------------
# What marl_debug_tail_run builds itself and a learner builds from its handle: the sums-of-squares buffer and grads_are_local (fused tail and the
# two-kernel fallback of marl_dqn_update, path 0 / 1, against marl_dqn_update_grads + _update_apply, path 2), the tensor-core images the step keeps
# current, and the actor-critic's critic-only target slice [n_actor, n_actor + n_critic).  Bars: the gradient against the oracle at the 1e-5 of
# every learner parity test; the norm, the step and the targets against tail_ref from the device's own gradient, with the kernel-level bars above.
def _learner_step_checks(where, path, n, shape, met, g, theta0, m0, v0, tgt0, theta, m, v, tgt, grad_clip, step, target, tau):
    gd, sd = g[:n].astype(np.float64), g[n:n + 4].astype(np.float64)
    norm_d = math.sqrt(float((gd * gd).sum())) / sd[1]
    _note("learner: norm", abs(float(met[1]) - norm_d) / (tr.norm_bar(path, n, shape) * norm_d), where)
    dclip = tr.device_clip(met[1], grad_clip)
    ref = tr.step_ref(gd, sd, theta0, m0, v0, tgt0, "Adam", 3e-4, grad_clip, step, target, tau, clip=dclip)
    bars = tr.step_bars("Adam", ref, theta0, tgt0, tau, target)
    _note("learner: theta", tr.worst(theta, ref["theta"], bars["theta"]), where)
    _note("learner: m", tr.worst(m, ref["m"], bars["m"]), where)
    _note("learner: v", tr.worst(v, ref["v"], bars["v"]), where)
    mode, begin, count = target
    if mode == 1:
        assert np.array_equal(tgt, theta[begin:begin + count]), f"{where}: hard target is not the new theta"
    elif mode == 2:
        _note("learner: Polyak target", tr.worst(tgt, ref["tgt"][:count], bars["tgt"]), where)
    else:
        assert np.array_equal(tgt, tgt0), f"{where}: no target update was due, but theta_tgt changed"


def _dqn_images_equal_a_repack(m, ts, idx, obs, where):
    def outputs():
        q, tq = m.q_values(obs).clone(), m.q_values(obs, target=True).clone()
        m.update_grads(ts, idx)
        return dict(q=q.cpu(), target_q=tq.cpu(), grad=m.grad.cpu().clone())

    kept = outputs()
    m.params_changed()
    repacked = outputs()
    for k in kept:
        assert torch.equal(kept[k], repacked[k]), f"{where}: {k} from the images the step kept current differs from a full repack"


def _learner_labels():
    return ["pb=128 small edge", "refused below", "pb=512 top", "refused above"] + [f"pb={pb}" for pb in range(tr.MIN_PB, tr.MAX_PB + 1, 32)]


@pytest.mark.parametrize("label", _learner_labels())
def test_idqn_handle_tail(label):
    """One marl_dqn_update (the fused tail, or its two-kernel fallback around the refusals) and one marl_dqn_update_grads + _update_apply on an IDQN
    handle whose parameter count lands in `label`'s class on this device; Polyak targets on even classes, a hard sync at the second update on odd
    ones; for H = 128 the images the step kept current equal a full repack after each update."""
    import types

    from oracle import learner_ref as lr
    from tests import hidden_width_ref as hr
    from tests.helpers import assert_grad_close, random_store, redraw_on_near_tie, space, traj_store

    from codebase_b200.dqn import model as M

    cases = tr.learner_cases(CAP[1])
    if label not in cases:
        pytest.skip(f"no IDQN configuration of up to 4 networks lands in {label} at capacity {CAP[1]}")
    N, D, H, A, n = cases[label]
    shape = tr.tail_shape(n, CAP[1])
    assert (shape is None) == label.startswith("refused"), (label, n, shape)
    k = _learner_labels().index(label)
    tu = 0.05 if k % 2 == 0 else 2
    grad_clip = 1.0
    B, T, cap = 8, 6, 16

    @redraw_on_near_tie
    def body():
        cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=grad_clip, double_q=False, target_update_interval_or_tau=tu,
                                    standardise_returns=False)
        m = M.QNetwork([space(shape=(D,))] * N, [space(n=A)] * N, cfg, [H, H], False, False, True, "cuda", max_batch=B, max_episode_length=T)
        try:
            assert m.n_params == n
            m.theta_tgt.copy_(m.theta + 0.01 * torch.randn_like(m.theta)); m.params_changed()
            hp = lr.DqnHP(grad_clip=grad_clip, double_q=False, target_update_interval_or_tau=tu)
            rng = np.random.default_rng(n)
            store = random_store(rng, cap, N, T, D, False, A=A)
            ts = traj_store(store, m.device)
            obs = torch.tensor(rng.integers(-1, 12, size=(33, N, D)), dtype=torch.float32, device=m.device)
            for u, kind in enumerate(("update", "update_grads + update_apply")):
                where = f"IDQN {label} (N {N}, D {D}, H {H}, A {A}, n {n}) {kind}"
                theta0, m0, v0, tgt0 = (x.cpu().numpy().copy() for x in (m.theta, m.adam_m, m.adam_v, m.theta_tgt))
                idx = rng.integers(0, cap, size=B).astype(np.int32)
                batch = lr.batch_from_store(store, idx)
                st = lr.DqnState(torch.tensor(theta0), torch.tensor(tgt0), list(m.agent_net), D, A)
                with hr.networks([]):
                    want = lr.dqn_update(copy.deepcopy(st), batch, hp)
                didx = torch.tensor(idx, device=m.device)
                if kind == "update":
                    met = m.update_from_store(ts, didx).cpu().numpy().copy()
                    path = 1 if shape is None else 0
                else:
                    m.update_grads(ts, didx)
                    met = m.update_apply().cpu().numpy().copy()
                    path = 2
                g = m.grad.cpu().numpy().copy()
                _record_grad(g[:n] / g[n + 1], want["grad"].numpy(), where)
                with hr.networks([]):
                    assert_grad_close(lr, st, batch, hp, g[:n] / g[n + 1], want["grad"].numpy(), tol=1e-5, what=where)
                mode = 2 if tu < 1 else (1 if u + 1 >= tu else 0)
                _learner_step_checks(where, path, n, shape, met, g, theta0, m0, v0, tgt0, *(x.cpu().numpy() for x in (m.theta, m.adam_m, m.adam_v, m.theta_tgt)),
                                     grad_clip, u + 1, (mode, 0, n), tu)
                if H == 128:
                    _dqn_images_equal_a_repack(m, ts, didx, obs, where)
        finally:
            m.close()

    body()


@pytest.mark.parametrize("A", [4, 5, 6])
@pytest.mark.parametrize("tu", [2, 0.05])
def test_ia2c_handle_tail(A, tu):
    """IA2C (one agent, obs 10, hidden 128): n = n_actor + n_critic with n % 4 = 1, 2, 3 for A = 4, 5, 6 (adam_kernel's float4 norm and its scalar
    tail; n_actor is odd at A = 5), two updates at env steps 1 and 2: the critic-only target slice [n_actor, n) is hard-copied at step 2 (tu = 2) or
    moved by Polyak at both (tu = 0.05), the actor's parameters never reach theta_tgt."""
    from oracle import learner_ref as lr
    from tests.helpers import ac_batch, ac_model, ac_oracle_batch, assert_grad_close, redraw_on_near_tie, traj_store

    N, D, P, T = 1, 10, 8, 6
    na, nc = tr.ac_params(N, D, 128, A)
    n = na + nc
    assert n % 4 == (A - 3)

    @redraw_on_near_tie
    def body():
        hp = lr.A2CHP(grad_clip=0.5, target_update_interval_or_tau=tu)
        m = ac_model(hp, N, D, P, T, A=A)
        try:
            assert (m.n_actor, m.n_critic) == (na, nc)
            m.theta_tgt.copy_(m.theta_tgt + 0.01 * torch.randn_like(m.theta_tgt))
            rng = np.random.default_rng(A)
            for step in (1, 2):
                where = f"IA2C A {A} tu {tu} (n {n}, n_actor {na}) step {step}"
                theta0, m0, v0, tgt0 = (x.cpu().numpy().copy() for x in (m.theta, m.adam_m, m.adam_v, m.theta_tgt))
                st = lr.A2CState(torch.tensor(theta0[:na]), torch.tensor(theta0[na:]), torch.tensor(tgt0), list(m.actor_net), list(m.critic_net), D, A)
                s = ac_batch(rng, P, N, T, D, A)
                batch = ac_oracle_batch(s)
                want = lr.a2c_update(copy.deepcopy(st), batch, hp, step)
                met = m.update_from_store(traj_store(s, m.device), P, step).cpu().numpy().copy()
                g = m.grad.cpu().numpy().copy()
                raw = np.concatenate([want["grad"]["actor"].numpy(), want["grad"]["critic"].numpy()])
                _record_grad(g[:n] / g[n + 1], raw, where)
                assert_grad_close(lr, st, batch, hp, g[:n] / g[n + 1], raw, tol=1e-5, what=where, kink_risk=lambda: lr.a2c_kink_risk(st, batch, hp))
                mode = 2 if tu < 1 else (1 if step % tu == 0 else 0)
                _learner_step_checks(where, 2, n, None, met, g, theta0, m0, v0, tgt0, *(x.cpu().numpy() for x in (m.theta, m.adam_m, m.adam_v, m.theta_tgt)),
                                     0.5, step, (mode, na, nc), tu)
        finally:
            m.close()

    body()

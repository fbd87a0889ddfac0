"""GPU: the Huber TD loss of IDQN, VDN and QMIX (algorithm.huber_delta; td_error in csrc/dqn_heads.cuh, reached by the fused FP32 training kernel,
the tensor-core dH1 kernel, col_td_kernel and qmix_mix_kernel) against the float64 oracle (tests/huber_ref.py): loss, gradients and parameters after
each update of unglued chains on ragged episodes -- the tensor-core and the FP32 training pass, GRU agents, both QMIX mixers, double-Q on and off,
standardise_returns, td_lambda, truncated episodes, parameter sharing, stale tails -- with delta at the median |TD error| of the first batch, so both
sides of the band are taken; huber_delta = null against a handle that never heard of the option, bit for bit; the update_n chain against its loop
and the oracle; the ABI's refusals; the training drivers end to end; and two data-parallel ranks against one process on the same global batch."""
import copy
import ctypes as C
import dataclasses
import os
import signal
import socket
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from oracle import learner_ref as lr
from oracle import policy_ref
from oracle import qmix_ref as qr
from tests import hidden_width_ref as hw
from tests import huber_ref as hr
from tests import qmix_options_ref as qo
from tests.helpers import TIE, NearTie, assert_grad_close, random_store, redraw_on_near_tie, space, traj_store

pytestmark = pytest.mark.gpu
A = 6
MIXER = {"idqn": 0, "vdn": 1, "qmix": 2}
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@dataclasses.dataclass(frozen=True)
class Case:
    kind: str = "idqn"
    lam: float = None       # algorithm.td_lambda
    N: int = 2
    D: int = 9
    T: int = 25
    B: int = 16
    H: int = 128
    rnn: bool = False
    hl: int = 2
    sharing: bool = False
    double_q: bool = True
    standardise: bool = False
    tu: float = 2.0
    tails: str = "ragged"   # ragged: done before T, unfilled tails; truncated: no done flag at all (use_proper_termination); stale: filled again after a gap


def _hp(c):
    return lr.DqnHP(double_q=c.double_q, target_update_interval_or_tau=c.tu, mixer=MIXER[c.kind])


def _model(c, delta=1.0, with_key=True):
    """with_key False: a configuration without the huber_delta key at all"""
    from codebase_b200.dqn import model as M

    hp = _hp(c)
    cfg = types.SimpleNamespace(optimizer="Adam", lr=hp.lr, gamma=hp.gamma, grad_clip=hp.grad_clip, double_q=c.double_q, target_update_interval_or_tau=c.tu,
                                standardise_returns=c.standardise, td_lambda=c.lam)
    if with_key:
        cfg.huber_delta = delta
    obs, act = [space(shape=(c.D,))] * c.N, [space(n=A)] * c.N
    if c.kind == "qmix":
        return M.QMixNetwork(obs, act, cfg, [c.H, c.H], c.sharing, c.rnn, True, dict(embed_dim=32, hypernet_layers=c.hl, hypernet_embed=32), "cuda",
                             max_batch=c.B, max_episode_length=c.T)
    cls = M.VDNetwork if c.kind == "vdn" else M.QNetwork
    return cls(obs, act, cfg, [c.H, c.H], c.sharing, c.rnn, True, "cuda", max_batch=c.B, max_episode_length=c.T)


def _perturb_target(m):
    m.theta_tgt.copy_(m.theta + 0.01 * torch.randn_like(m.theta))
    if m.mixer == 2:
        m.mix_tgt.copy_(m.mix + 0.01 * torch.randn_like(m.mix))
    m.params_changed()


def _copy_params(a, b):
    for k in ("theta", "theta_tgt") + (("mix", "mix_tgt") if a.mixer == 2 else ()):
        getattr(b, k).copy_(getattr(a, k))
    b.params_changed()


def _agent_net(c):
    return [0] * c.N if c.sharing else list(range(c.N))


def _oracle(c, m):
    ms = (lambda: lr.RunningMeanStdRef((c.N,) if c.kind == "idqn" else (1,))) if c.standardise else (lambda: None)
    if c.kind == "qmix":
        return qo.QmixOptState(m.theta.cpu().clone(), m.theta_tgt.cpu().clone(), m.mix.cpu().clone(), m.mix_tgt.cpu().clone(), _agent_net(c), c.D, A,
                               embed_dim=32, hypernet_layers=c.hl, ret_ms=ms())
    return lr.DqnState(m.theta.cpu().clone(), m.theta_tgt.cpu().clone(), _agent_net(c), c.D, A, ret_ms=ms())


def _store(c, seed, cap=None):
    """cap episodes (default B) in the device layout, rewards spread over [0, 4); VDN and QMIX see the team reward"""
    rng = np.random.default_rng(seed)
    s = random_store(rng, cap or c.B, c.N, c.T, c.D, c.kind != "idqn", A=A)
    s["rew"] *= 4.0
    if c.tails == "truncated":
        s["done"][:] = 0
    elif c.tails == "stale":
        for e in range(0, s["filled"].shape[0], 2):
            L = int(s["filled"][e].sum())
            if L + 1 < c.T:
                s["filled"][e, L + 1:] = 1
                s["done"][e, L + 1:] = rng.random(c.T - L) < 0.2
    return s


def _nets(c):
    return hw.networks({(c.D, A)} if c.rnn else ())


def _median_delta(c, st, batch, hp):
    """delta at the median |TD error| over the filled rows of the batch (rounded to 3 significant digits): both branches taken"""
    with _nets(c):
        if c.kind == "qmix":
            d = hr.qmix_td(st.theta, st.mix, dataclasses.replace(st, ret_ms=copy.deepcopy(st.ret_ms)), batch, hp, c.lam)
        else:
            d = hr.dqn_td(st.theta, st.theta_tgt, st.agent_net, c.D, A, batch, hp, copy.deepcopy(st.ret_ms), c.lam)
    m = batch["filled"].double().expand_as(d) > 0
    delta = float(np.format_float_positional(float(d.detach().abs()[m].median()), precision=3, unique=False, fractional=False))
    inside, outside = hr.branches(d, batch["filled"], delta)
    assert inside > 0 and outside > 0, (inside, outside)
    return delta


def _update_oracle(c, st, batch, hp, delta):
    with _nets(c), hr.huber_in(delta, c.lam):
        return qr.qmix_update(st, batch, hp) if c.kind == "qmix" else lr.dqn_update(st, batch, hp)


def _margin(c, st, batch, hp):
    if not c.double_q:
        return
    with _nets(c):
        margin = lr.double_q_margin(lr.DqnState(st.theta, st.theta_tgt, st.agent_net, c.D, A), batch, hp)
    if margin < TIE:
        raise NearTie(f"double-Q argmax margin {margin:.1e}")


def _kink(c, st0, batch, hp, delta):
    def risk():
        with _nets(c):
            if c.kind == "qmix":
                return hr.qmix_kink_risk(st0, batch, hp, delta, c.lam)
            with hr.huber_in(delta, c.lam):
                return lr.dqn_kink_risk(st0, batch, hp)
    return risk


def _close(got, want, tol, what):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    scale = max(1.0, float(np.abs(want).max()))
    err = float(np.abs(got - want).max())
    assert err <= tol * scale, f"{what}: max abs error {err:.3e} > {tol:g} x {scale:.3g}"


def _check_update(c, m, st, st0, batch, want, met, hp, delta, what):
    filled = float(batch["filled"].sum())
    assert abs(float(met[0]) - want["loss"]) <= 1e-5 * max(1.0, abs(want["loss"])), f"loss {float(met[0])} vs {want['loss']}, {what}"
    assert_grad_close(lr, st0, batch, hp, m.grad[: m.n_params].cpu().numpy() / filled, want["grad"].numpy(), tol=1e-5, what=f"agents' gradient, {what}",
                      kink_risk=_kink(c, st0, batch, hp, delta))
    mine = [(m.theta, st.theta, "theta"), (m.theta_tgt, st.theta_tgt, "target")]
    if c.kind == "qmix":
        _close(m.mix_grad[: m.n_mix].cpu().numpy() / filled, want["mix_grad"].numpy(), 1e-5, f"mixer gradient, {what}")
        mine += [(m.mix, st.mix, "mixer"), (m.mix_tgt, st.mix_tgt, "target mixer")]
    for got, ref, name in mine:
        assert np.quantile(np.abs(got.cpu().numpy() - ref.numpy()), 0.999) < 1e-5, f"{name} after {what}"
    if c.standardise:
        mean, var, count = m.ret_ms()
        want_mean, want_var = np.broadcast_to(st.ret_ms.mean.numpy(), mean.shape), np.broadcast_to(st.ret_ms.var.numpy(), var.shape)
        np.testing.assert_allclose(mean.numpy(), want_mean, rtol=1e-5, atol=1e-6, err_msg=f"ret_ms mean, {what}")
        np.testing.assert_allclose(var.numpy(), want_var, rtol=1e-5, atol=1e-5, err_msg=f"ret_ms var, {what}")
        assert count == pytest.approx(st.ret_ms.count, rel=1e-12), what


def _run_chain(c, n_updates=3):
    hp = _hp(c)
    m = _model(c)
    assert m.huber_delta == 1.0
    _perturb_target(m)
    st = _oracle(c, m)
    idx = torch.arange(c.B, dtype=torch.int32, device=m.device)
    delta = None
    for u in range(n_updates):
        s = _store(c, 1000 * u + c.B + c.T)
        batch = lr.batch_from_store(s, np.arange(c.B))
        _margin(c, st, batch, hp)
        if delta is None:
            delta = _median_delta(c, st, batch, hp)
            m.set_huber_delta(delta)
        st0 = copy.deepcopy(st)
        want = _update_oracle(c, st, batch, hp, delta)
        met = m.update_from_store(traj_store(s, m.device), idx).cpu()
        _check_update(c, m, st, st0, batch, want, met, hp, delta, f"update {u}, delta {delta}")
    m.close()


# ---- 1. unglued chains against the oracle --------------------------------------------------------------------------------------------------------
CHAIN = {
    "idqn_tc": Case(),
    "idqn_tc_single_q_truncated": Case(double_q=False, tails="truncated"),
    "idqn_tc_standardise_polyak": Case(standardise=True, tu=0.05),
    "idqn_tc_shared_stale": Case(sharing=True, tails="stale", N=3),
    "idqn_tc_lam0": Case(lam=0.0),
    "idqn_tc_lam06_standardise": Case(lam=0.6, standardise=True),
    "idqn_tc_d32": Case(D=32),   # observations of 32 features: the FP32 training pass with the 128-wide network
    "idqn_fp32": Case(H=64),
    "idqn_fp32_shared_single_q": Case(H=64, sharing=True, double_q=False, N=3),
    "idqn_fp32_lam06_stale": Case(H=64, lam=0.6, tails="stale"),
    "vdn_tc": Case(kind="vdn", N=3),
    "vdn_tc_standardise": Case(kind="vdn", standardise=True),
    "vdn_tc_single_q_truncated_lam06": Case(kind="vdn", double_q=False, tails="truncated", lam=0.6),
    "vdn_d32": Case(kind="vdn", D=32),
    "vdn_fp32_shared": Case(kind="vdn", H=64, sharing=True),
    "qmix_h2": Case(kind="qmix"),
    "qmix_h1": Case(kind="qmix", hl=1, N=3),
    "qmix_h1_standardise_lam0": Case(kind="qmix", hl=1, standardise=True, lam=0.0),
    "qmix_h2_lam06_stale": Case(kind="qmix", lam=0.6, tails="stale"),
    "qmix_h2_single_q_shared_truncated": Case(kind="qmix", double_q=False, sharing=True, tails="truncated", tu=0.05),
    "rnn_idqn": Case(rnn=True, T=9, B=8),
    "rnn_idqn_standardise_lam06": Case(rnn=True, T=9, B=8, standardise=True, lam=0.6),
    "rnn_vdn_stale": Case(kind="vdn", rnn=True, T=9, B=8, tails="stale"),
    "rnn_qmix_h1": Case(kind="qmix", hl=1, rnn=True, T=9, B=8),
}


@pytest.mark.parametrize("name", list(CHAIN))
@redraw_on_near_tie
def test_unglued_chain_matches_oracle(name):
    """three updates through marl_dqn_update on fresh ragged batches; the device state is never re-synchronised with the oracle"""
    _run_chain(CHAIN[name])


# ---- 2. huber_delta = null is the squared error, bit for bit --------------------------------------------------------------------------------------
NULL = {"idqn_tc": Case(), "idqn_tc_standardise": Case(standardise=True), "idqn_tc_lam06": Case(lam=0.6), "idqn_d32": Case(D=32),
        "idqn_fp32": Case(H=64), "vdn": Case(kind="vdn"), "vdn_fp32": Case(kind="vdn", H=64), "qmix_h1": Case(kind="qmix", hl=1),
        "qmix_h2_standardise": Case(kind="qmix", standardise=True), "rnn_idqn": Case(rnn=True, T=9, B=8),
        "rnn_qmix_h2": Case(kind="qmix", rnn=True, T=9, B=8)}


def _state(m):
    out = dict(theta=m.theta, theta_tgt=m.theta_tgt, adam_m=m.adam_m, adam_v=m.adam_v, grad=m.grad, metrics=m._metrics)
    if m.mixer == 2:
        out.update(mix=m.mix, mix_tgt=m.mix_tgt, mix_m=m.mix_m, mix_v=m.mix_v, mix_grad=m.mix_grad)
    return {k: v.detach().cpu().clone() for k, v in out.items()}


def _assert_same(a, b, what):
    got, ref = _state(a), _state(b)
    for k in ref:
        assert torch.equal(got[k], ref[k]), f"{k}, {what}: max abs difference {float((got[k].double() - ref[k].double()).abs().max()):.3e}"


@pytest.mark.parametrize("name", list(NULL))
def test_null_delta_is_bit_identical_to_no_setter(name):
    """a handle configured with huber_delta: null, and one switched to Huber and back with set_huber_delta(None), against a handle whose
    configuration has no huber_delta key (the setter is never called): parameters, Adam state, gradient and loss equal after every update"""
    c = NULL[name]
    a, b, x = _model(c, delta=None), _model(c, with_key=False), _model(c, delta=0.5)
    assert a.huber_delta is None and b.huber_delta is None
    _perturb_target(b)
    _copy_params(b, a); _copy_params(b, x)
    x.set_huber_delta(None)
    idx = torch.arange(c.B, dtype=torch.int32, device=a.device)
    for u in range(3):
        ts = traj_store(_store(c, 40 + u), a.device)
        for m in (a, b, x):
            m.update_from_store(ts, idx)
        _assert_same(a, b, f"null, update {u}")
        _assert_same(x, b, f"switched off, update {u}")
    a.close(); b.close(); x.close()


# ---- 3. update_n: the loop it replaces, bit for bit, and the oracle ------------------------------------------------------------------------------
SEED = 0x4B7E


@pytest.mark.parametrize("kind", ["idqn", "vdn", "qmix"])
@redraw_on_near_tie
def test_update_n_is_the_loop_it_replaces_and_tracks_the_oracle(kind):
    from codebase_b200 import _native as nat

    c, K, cap, delta = Case(kind=kind, T=12, B=24, tu=3.0), 4, 64, 0.3
    hp = _hp(c)
    a, b = _model(c, delta), _model(c, delta)
    _perturb_target(a)
    _copy_params(a, b)
    st = _oracle(c, a)
    s = _store(c, 77, cap)
    ts = traj_store(s, a.device)
    a.update_n(ts, c.B, cap, SEED, 0, K)
    idx = torch.zeros(c.B, dtype=torch.int32, device=b.device)
    for u in range(K):
        nat.check(nat.lib().marl_replay_sample(C.c_uint64(SEED), C.c_uint64(u), C.c_int32(c.B), C.c_int32(cap), nat.ptr(idx), nat.stream_ptr()), "marl_replay_sample")
        ids = policy_ref.replay_sample(SEED, u, c.B, cap)
        assert np.array_equal(idx.cpu().numpy(), ids), f"replay indices of update {u}"
        batch = lr.batch_from_store(s, ids)
        _margin(c, st, batch, hp)
        st0 = copy.deepcopy(st)
        want = _update_oracle(c, st, batch, hp, delta)
        met = b.update_from_store(ts, idx).cpu()
        _check_update(c, b, st, st0, batch, want, met, hp, delta, f"update {u}")
    _assert_same(a, b, "update_n against its loop")
    assert a.updates == b.updates == K
    a.close(); b.close()


# ---- 4. the ABI ------------------------------------------------------------------------------------------------------------------------------------
def test_abi_refuses_a_bad_delta_on_a_live_handle():
    from codebase_b200 import _native as nat

    m = _model(Case(), delta=None)
    for bad in (0.0, -1.0, float("nan"), float("inf")):
        rc = nat.lib().marl_dqn_set_huber_delta(m._h, C.c_int32(1), C.c_float(bad))
        assert rc < 0 and b"finite number > 0" in nat.lib().marl_last_error(), bad
    assert nat.lib().marl_dqn_set_huber_delta(m._h, C.c_int32(1), C.c_float(0.5)) == 0
    assert nat.lib().marl_dqn_set_huber_delta(m._h, C.c_int32(0), C.c_float(float("nan"))) == 0
    with pytest.raises(ValueError, match="huber_delta"):
        m.set_huber_delta(-2.0)
    m.close()


# ---- 5. the drivers -------------------------------------------------------------------------------------------------------------------------------
DRIVER_COLS = ["environment_steps", "agent0/mean_episode_returns", "agent0/std_episode_returns", "agent1/mean_episode_returns", "agent1/std_episode_returns",
               "epsilon", "loss", "mean_episode_length", "mean_episode_returns", "mean_episode_time", "std_episode_length", "std_episode_returns",
               "std_episode_time", "updates"]


@pytest.mark.parametrize("alg,env,extra", [
    ("idqn", "lbforaging:Foraging-8x8-2p-3f-v3", []),
    ("vdn", "matrixgames:penalty-100-nostate-v0", ["algorithm.use_proper_termination=True"]),
    ("qmix", "matrixgames:penalty-100-nostate-v0", []),
    ("qmix", "lbforaging:Foraging-8x8-2p-3f-v3", ["algorithm.model.mixing.hypernet_layers=1", "algorithm.td_lambda=0.6"]),
])
def test_driver_with_huber_delta(tmp_path, monkeypatch, alg, env, extra):
    import pandas as pd

    from codebase_b200 import run

    monkeypatch.chdir(tmp_path)
    run.main([f"+algorithm={alg}", f"env.name={env}", "env.time_limit=25", "env.parallel_envs=256", "seed=0",
              "algorithm.total_steps=60000", "algorithm.eval_interval=20000", "algorithm.batch_size=128", "algorithm.buffer_size=4096",
              "algorithm.updates_per_iteration=16", "algorithm.huber_delta=1.0", f"run_dir={tmp_path}/out"] + extra)
    df = pd.read_csv(tmp_path / "out" / "results.csv")
    assert list(df.columns) == DRIVER_COLS
    assert len(df) >= 2 and df["updates"].iloc[-1] > 0 and np.isfinite(df["loss"][df["updates"] > 0]).all()


# ---- 6. two data-parallel ranks on one device against one process ---------------------------------------------------------------------------------
DP_SCRIPT = r"""
import sys, types
import numpy as np, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
from codebase_b200.dqn import model as M
from tests.helpers import random_store, space, traj_store
kind, out = sys.argv[2], sys.argv[3]
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
torch.cuda.set_device(0)
N, D, T, B, A = 2, 9, 12, 32, 6
cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=1.0, double_q=True, target_update_interval_or_tau=2.0,
                            standardise_returns=False, td_lambda=None, huber_delta=0.3)
obs, act = [space(shape=(D,))] * N, [space(n=A)] * N
B_local = B // world
torch.manual_seed(5)
if kind == "qmix":
    m = M.QMixNetwork(obs, act, cfg, [128, 128], False, False, True, dict(embed_dim=32, hypernet_layers=2, hypernet_embed=32), "cuda", max_batch=B_local, max_episode_length=T)
else:
    m = M.QNetwork(obs, act, cfg, [128, 128], False, False, True, "cuda", max_batch=B_local, max_episode_length=T)
s = random_store(np.random.default_rng(11), B, N, T, D, kind != "idqn", A=A)
s["rew"] *= 4.0
ts = traj_store(s, m.device)
losses = []
for u in range(3):
    idx = torch.arange(rank * B_local, (rank + 1) * B_local, dtype=torch.int32, device=m.device)
    m.update_grads(ts, idx)
    for t in m.exchanged_buffers():
        host = t.cpu()
        dist.all_reduce(host)
        t.copy_(host.to(t.device))
    losses.append(float(m.update_apply()[0]))
    s["rew"] = np.roll(s["rew"], 1, axis=2)
    ts = traj_store(s, m.device)
if rank == 0:
    res = dict(loss=np.array(losses), theta=m.theta.cpu().numpy())
    if kind == "qmix":
        res["mix"] = m.mix.cpu().numpy()
    np.savez(out, **res)
dist.destroy_process_group()
"""


@pytest.mark.parametrize("kind", ["idqn", "qmix"])
def test_two_ranks_match_one_process(tmp_path, kind):
    """with delta set, two torchrun ranks on one device (each half the global batch, gradient buffers summed over gloo) give the loss and the
    parameters of one process on the whole batch"""
    script = tmp_path / "dp.py"
    script.write_text(DP_SCRIPT)
    outs = {}
    for world in (1, 2):
        out = tmp_path / f"w{world}.npz"
        with socket.socket() as sk:
            sk.bind(("127.0.0.1", 0))
            port = sk.getsockname()[1]
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", f"--master-port={port}", str(script), ROOT, kind, str(out)]
        p = subprocess.Popen(cmd, cwd=str(tmp_path), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, start_new_session=True)
        try:
            log, _ = p.communicate(timeout=600)
        finally:
            if p.poll() is None:
                os.killpg(p.pid, signal.SIGKILL)
                p.communicate()
        assert p.returncode == 0, log.decode(errors="replace")[-4000:]
        outs[world] = np.load(out)
    one, two = outs[1], outs[2]
    np.testing.assert_allclose(two["loss"], one["loss"], rtol=1e-5, atol=1e-6)
    for k in ("theta",) + (("mix",) if kind == "qmix" else ()):
        assert np.quantile(np.abs(two[k] - one[k]), 0.999) < 1e-5, k
